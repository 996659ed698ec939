// TEST INFRASTRUCTURE: the oracle twin of the kafka workload (MS_W_KAFKA, DESIGN.md 2.15), written apart from the
// device code (csrc/ms_raft.cuh kf_handle, csrc/ms_kernels.cu kf_gen_step).
//
// It is the CPU oracle (oracle/oracle.cpp, compiled into this unit as it is) plus the single-node kafka node of
// demo/clojure/kafka_single_node.clj and the Client of workload/kafka.clj:191-241 with the generator of the engine's
// header (ms_add_kafka_clients).  The node keeps maps of vectors, the client a map of offsets, as the reference does.
// The round loop below restates or_sim::run_round for what a kafka simulation contains: the injector, the nodes,
// host-visible clients, client sinks and the kafka clients.  Send, queues, the journal and time are the oracle's.
//
//     g++ -O2 -std=c++17 -fPIC -shared tests/native/kafka_oracle.cpp -o tests/native/_build/libkafka_oracle.so
#include <map>

#include "../../oracle/oracle.cpp"

extern "C" {
typedef struct orkf_config {          // the engine's ms_kafka_gen_config, restated
  uint32_t n_clients, assign_permille, crash_permille, pad;
  int64_t  interval_ns, timeout_ns, time_limit_ns;
} orkf_config;
typedef struct orkf_hist {            // the engine's ms_kafka_hist, restated
  int64_t  time_ns;
  uint64_t order;
  uint32_t client, op;
  uint8_t  type, f;
  uint16_t error;
  uint32_t key[2], a[2], b[2];
  uint32_t pad[3];
} orkf_hist;
}

namespace {
enum { T_SEND = 70, T_SEND_OK = 71, T_POLL = 72, T_POLL_OK = 73, T_COMMIT = 74, T_COMMIT_OK = 75, T_LIST = 76,
       T_LIST_OK = 77 };
enum { HF_SEND = 10, HF_POLL = 11, HF_ASSIGN = 12, HF_CRASH = 13 };
enum { H_INVOKE = 0, H_OK = 1, H_FAIL = 2, H_INFO = 3 };
constexpr uint32_t kNoKey = 0xFFFF, kNone = 0xFFFFFFFFu;

struct KafkaNode {                                   // the atoms of kafka_single_node.clj
  std::map<uint32_t, std::vector<uint32_t>> queues;  // key -> messages (:150-153)
  std::map<uint32_t, uint32_t> committed;            // key -> committed offset (:155-157)
};

struct Slot { uint32_t key = kNoKey, a = 0, b = 0; };
struct KafkaClient {                                 // Client (workload/kafka.clj:191-241)
  std::vector<uint32_t> assigned;                    // the assignment, in the order it was drawn
  std::map<uint32_t, uint32_t> offsets;              // `offsets`: key -> the offset to read next
  enum { IDLE, LIST, SEND, POLL, COMMIT } waiting = IDLE;
  uint32_t sends = 0;
  Slot slot[2];                                      // the history slots of the op in flight
  std::vector<uint32_t> assigning;                   // assign: the keys drawn
};

std::pair<uint32_t, uint32_t> keys_of(uint32_t p0) { return {p0 & 0xFFFF, p0 >> 16}; }
}  // namespace

struct orkf {
  or_sim* s;
  uint32_t n_keys, log_cap;
  std::vector<KafkaNode> nodes;
  orkf_config cfg{};
  uint32_t first = 0;
  std::vector<KafkaClient> clients;                  // by ordinal
  std::vector<orkf_hist> hist;
  size_t drained = 0;

  bool key_ok(uint32_t k) {
    if (k == kNoKey || k < n_keys) return true;
    s->error = "kafka oracle: key out of range";
    return false;
  }

  // process-stdin!'s future for one message (:121-146) and the handlers (:159-207)
  void node(uint32_t e, const or_msg& m, std::vector<Emit>& out) {
    if (m.flags & OR_F_REPLY) return;                                  // handle-reply!: rpcs is empty
    KafkaNode& nd = nodes[e];
    or_msg a; std::memset(&a, 0, sizeof a);
    a.src = e; a.dest = m.src;
    if (m.flags & OR_F_MSG_ID) { a.flags = OR_F_REPLY; a.in_reply_to = m.msg_id; }   // reply!
    auto [k0, k1] = keys_of(m.p0);
    const uint32_t ks[2] = {k0, k1}, os[2] = {(uint32_t)m.p1, (uint32_t)(m.p1 >> 32)};
    if (m.type == OR_T_INIT) {
      a.type = OR_T_INIT_OK;
    } else if (m.type == T_SEND) {
      if (m.p0 >= n_keys) { s->error = "kafka oracle: key out of range"; return; }
      std::vector<uint32_t>& q = nd.queues[m.p0];
      if (q.size() >= log_cap) { s->error = "kafka oracle: log full"; return; }
      q.push_back((uint32_t)m.p1);
      a.type = T_SEND_OK;
      a.p1 = q.size() - 1;
    } else if (m.type == T_POLL) {
      if (!key_ok(k0) || !key_ok(k1)) return;
      uint32_t keys[2] = {kNoKey, kNoKey};
      for (int i = 0; i < 2; i++) {
        if (ks[i] == kNoKey) continue;
        auto it = nd.queues.find(ks[i]);
        const uint32_t count = it == nd.queues.end() ? 0 : (uint32_t)it->second.size();
        if (std::min(os[i], count) == count) continue;                 // (subvec queue offset) is empty: omitted
        keys[i] = ks[i];
        a.p1 |= (uint64_t)count << (32 * i);
      }
      a.type = T_POLL_OK;
      a.p0 = keys[0] | (keys[1] << 16);
    } else if (m.type == T_COMMIT) {
      if (!key_ok(k0) || !key_ok(k1)) return;
      for (int i = 0; i < 2; i++) {
        if (ks[i] == kNoKey) continue;
        if (os[i] == kNone) { s->error = "kafka oracle: offset out of range"; return; }
        auto it = nd.committed.find(ks[i]);
        if (it == nd.committed.end()) nd.committed[ks[i]] = os[i];
        else it->second = std::max(it->second, os[i]);
      }
      a.type = T_COMMIT_OK;
    } else if (m.type == T_LIST) {
      if (!key_ok(k0) || !key_ok(k1)) return;
      uint32_t keys[2] = {kNoKey, kNoKey};
      for (int i = 0; i < 2; i++) {
        auto it = nd.committed.find(ks[i]);
        if (ks[i] == kNoKey || it == nd.committed.end()) continue;
        keys[i] = ks[i];
        a.p1 |= (uint64_t)it->second << (32 * i);
      }
      a.type = T_LIST_OK;
      a.p0 = keys[0] | (keys[1] << 16);
    } else {
      a.type = OR_T_ERROR;
      a.p0 = 10;
    }
    out.push_back(Emit(a));
  }

  void record(uint32_t e, uint8_t type, uint16_t err) {
    const Endpoint::Gen& g = s->eps[e].gen;
    const KafkaClient& c = clients[g.ordinal];
    orkf_hist h; std::memset(&h, 0, sizeof h);
    h.time_ns = s->now; h.order = (s->round << 24) | g.ordinal; h.client = e; h.op = g.ops;
    h.type = type; h.f = (uint8_t)g.cur_f; h.error = err;
    for (int i = 0; i < 2; i++) { h.key[i] = c.slot[i].key; h.a[i] = c.slot[i].a; h.b[i] = c.slot[i].b; }
    hist.push_back(h);
  }

  static void reopen(KafkaClient& c) { c.assigned.clear(); c.offsets.clear(); }   // a new Client (open!)

  or_msg request(uint32_t e, uint16_t type, uint32_t p0, uint64_t p1) {
    Endpoint::Gen& g = s->eps[e].gen;
    g.waiting_for = ++g.next_msg_id;
    g.deadline_ns = s->now + cfg.timeout_ns;
    or_msg m; std::memset(&m, 0, sizeof m);
    m.src = e; m.dest = g.node; m.type = type; m.flags = OR_F_MSG_ID; m.msg_id = g.waiting_for; m.p0 = p0; m.p1 = p1;
    return m;
  }

  // a reply delivered to client e: only the awaited id counts (client.clj:106-107)
  void reply(uint32_t e, const or_msg& m, std::vector<Emit>& out) {
    Endpoint::Gen& g = s->eps[e].gen;
    KafkaClient& c = clients[g.ordinal];
    if (!(m.flags & OR_F_REPLY) || g.waiting_for == 0 || m.in_reply_to != g.waiting_for) return;
    g.waiting_for = 0;
    if (m.type == OR_T_ERROR) {                                        // with-errors #{:assign}
      const bool indefinite = (m.p0 == 0 || m.p0 == 13) && c.waiting != KafkaClient::LIST;
      record(e, indefinite ? H_INFO : H_FAIL, (uint16_t)m.p0);
      if (indefinite) reopen(c);
      c.waiting = KafkaClient::IDLE;
      return;
    }
    auto [r0, r1] = keys_of(m.p0);
    const uint32_t rk[2] = {r0, r1}, rv[2] = {(uint32_t)m.p1, (uint32_t)(m.p1 >> 32)};
    switch (c.waiting) {
      case KafkaClient::LIST: {                                        // :assign (:204-219)
        std::map<uint32_t, uint32_t> committed, next;
        for (int i = 0; i < 2; i++) if (rk[i] != kNoKey) committed[rk[i]] = rv[i];
        for (size_t i = 0; i < c.assigning.size(); i++) {
          const uint32_t k = c.assigning[i];
          const auto lo = c.offsets.find(k);
          const auto co = committed.find(k);
          next[k] = lo != c.offsets.end() ? lo->second : co != committed.end() ? co->second : 0;
          c.slot[i] = Slot{k, next[k], co != committed.end() ? co->second : kNone};
        }
        c.offsets = next;
        c.assigned = c.assigning;
        record(e, H_OK, 0);
        c.waiting = KafkaClient::IDLE;
        break;
      }
      case KafkaClient::SEND:
        c.slot[0].b = rv[0];
        record(e, H_OK, 0);
        c.waiting = KafkaClient::IDLE;
        break;
      case KafkaClient::POLL: {                                        // apply-mop! :poll, then txn-offsets
        std::map<uint32_t, uint32_t> highest;
        for (int i = 0; i < 2; i++) {
          if (rk[i] == kNoKey) { c.slot[i] = Slot{}; continue; }
          c.slot[i] = Slot{rk[i], c.slot[i].a, rv[i]};                 // messages [a, b): the highest is b - 1
          highest[rk[i]] = rv[i] - 1;
          c.offsets[rk[i]] = std::max(c.offsets[rk[i]], rv[i]);        // merge-with max of (inc highest)
        }
        if (highest.empty()) { record(e, H_OK, 0); c.waiting = KafkaClient::IDLE; break; }
        uint32_t keys[2] = {kNoKey, kNoKey};
        uint64_t offs = 0;
        for (int i = 0; i < 2; i++)
          if (rk[i] != kNoKey) { keys[i] = rk[i]; offs |= (uint64_t)highest[rk[i]] << (32 * i); }
        c.waiting = KafkaClient::COMMIT;
        out.push_back(Emit(request(e, T_COMMIT, keys[0] | (keys[1] << 16), offs)));
        break;
      }
      default:                                                          // commit_offsets_ok: the poll is done
        record(e, H_OK, 0);
        c.waiting = KafkaClient::IDLE;
    }
  }

  // after the replies of the round: the timeout, then at most one invocation
  void step(uint32_t e, std::vector<Emit>& out) {
    Endpoint::Gen& g = s->eps[e].gen;
    KafkaClient& c = clients[g.ordinal];
    const int64_t now = s->now;
    if (g.waiting_for) {
      if (now < g.deadline_ns) return;
      const bool info = c.waiting != KafkaClient::LIST;
      record(e, info ? H_INFO : H_FAIL, 0xFFFF);
      if (info) reopen(c);
      c.waiting = KafkaClient::IDLE;
      g.waiting_for = 0;
    }
    if (g.phase != 0) return;
    if (now >= cfg.time_limit_ns) { g.phase = 3; return; }
    if (now < g.next_op_ns) return;
    const uint32_t ctr[4] = {g.ops, e, 0xC11E47u, 0u};
    const uint32_t key[2] = {s->cfg.seed_lo, s->cfg.seed_hi};
    uint32_t x[4];
    philox(ctr, key, x);
    g.next_op_ns = now + (int64_t)(((unsigned __int128)x[1] * (unsigned __int128)(2 * (uint64_t)cfg.interval_ns)) >> 32);
    g.ops++;
    const uint32_t r = (uint32_t)(((uint64_t)x[0] * 1000u) >> 32);
    const uint32_t k0 = (uint32_t)(((uint64_t)x[2] * n_keys) >> 32);
    c.slot[0] = c.slot[1] = Slot{};
    if (r < cfg.assign_permille) {
      g.cur_f = HF_ASSIGN;
      c.assigning = {k0};
      if (n_keys >= 2 && (x[3] & 1)) c.assigning.push_back((k0 + 1 + (uint32_t)(((uint64_t)x[3] * (n_keys - 1)) >> 32)) % n_keys);
      for (size_t i = 0; i < c.assigning.size(); i++) c.slot[i].key = c.assigning[i];
      record(e, H_INVOKE, 0);
      c.waiting = KafkaClient::LIST;
      const uint32_t k1 = c.assigning.size() > 1 ? c.assigning[1] : kNoKey;
      out.push_back(Emit(request(e, T_LIST, k0 | (k1 << 16), 0)));
    } else if (r < cfg.assign_permille + cfg.crash_permille) {
      g.cur_f = HF_CRASH;
      record(e, H_INVOKE, 0);
      record(e, H_INFO, 0);
      reopen(c);
    } else if (!(x[3] & 1)) {
      g.cur_f = HF_SEND;
      const uint32_t msg = g.ordinal + cfg.n_clients * c.sends++;
      c.slot[0] = Slot{k0, msg, kNone};
      record(e, H_INVOKE, 0);
      c.waiting = KafkaClient::SEND;
      out.push_back(Emit(request(e, T_SEND, k0, msg)));
    } else {
      g.cur_f = HF_POLL;
      uint32_t keys[2] = {kNoKey, kNoKey};
      uint64_t offs = 0;
      for (size_t i = 0; i < c.assigned.size(); i++) {
        keys[i] = c.assigned[i];
        c.slot[i] = Slot{keys[i], c.offsets[keys[i]], 0};
        offs |= (uint64_t)c.offsets[keys[i]] << (32 * i);
      }
      record(e, H_INVOKE, 0);
      c.waiting = KafkaClient::POLL;
      out.push_back(Emit(request(e, T_POLL, keys[0] | (keys[1] << 16), offs)));
    }
  }

  // or_sim::run_round's four steps (injector, endpoints in index order, visibility, time)
  bool round() {
    or_sim& o = *s;
    std::vector<Envelope> pending;
    uint32_t inj = 0;
    while (!o.host_queue.empty()) {
      or_msg m = o.host_queue.front(); o.host_queue.pop_front();
      if (!o.send(kInjector, inj++, m, pending)) return false;
    }
    while (o.sched_cursor < o.schedule.size() && o.schedule[o.sched_cursor].time_ns <= o.now) {
      const or_op& op = o.schedule[o.sched_cursor++];
      or_msg m; std::memset(&m, 0, sizeof m);
      m.src = op.src; m.dest = op.dest; m.type = op.body.type; m.flags = op.body.flags;
      m.msg_id = op.body.msg_id; m.in_reply_to = op.body.in_reply_to;
      m.p0 = op.body.p0; m.p1 = op.body.p1;
      if (!o.send(kInjector, inj++, m, pending)) return false;
    }
    std::vector<Emit> out;
    for (uint32_t e = 0; e < o.eps.size(); e++) {
      Endpoint& ep = o.eps[e];
      if (!ep.live) continue;
      out.clear();
      while (!ep.q.empty() && ep.q.top().m.deadline_ns <= o.now) {
        const or_msg m = ep.q.top().m;
        ep.q.pop();
        if (o.partitioned(m.src, e)) continue;
        o.log_event(true, m);
        switch (ep.kind) {
          case OR_KIND_CLIENT: case OR_KIND_HOST: ep.mailbox.push_back(m); break;
          case OR_KIND_SIM_CLIENT: if (m.flags & OR_F_REPLY) o.client_replies++; break;
          case OR_KIND_GEN_CLIENT: reply(e, m, out); break;
          case OR_KIND_SERVER: node(e, m, out); break;
          default: o.error = "kafka oracle: no services here"; return false;
        }
        if (!o.error.empty()) return false;
      }
      if (ep.kind == OR_KIND_GEN_CLIENT) step(e, out);
      for (uint32_t j = 0; j < out.size(); j++)
        if (!o.send(e, j, out[j].m, pending)) return false;
    }
    bool due_now = false;
    for (const Envelope& env : pending) {
      if (env.m.deadline_ns <= o.now) due_now = true;
      o.eps[env.m.dest].q.push(env);
    }
    o.round++;
    if (!due_now) o.now += kTickNs;
    return true;
  }

  bool stalled(int64_t& stall_now, uint64_t& stall_round) {
    if (s->now != stall_now) { stall_now = s->now; stall_round = s->round; return false; }
    if (s->round - stall_round > (1ull << 20)) { s->error = "virtual time is not advancing"; return true; }
    return false;
  }
};

extern "C" {

// The kafka nodes of a fresh oracle made with workload 7 and n_nodes servers: n_keys keys of log_cap messages each.
orkf* orkf_new(or_sim* s, uint32_t n_keys, uint32_t log_cap) {
  orkf* k = new orkf();
  k->s = s;
  k->n_keys = n_keys ? n_keys : 16;
  k->log_cap = log_cap ? log_cap : 4096;
  k->nodes.resize(s->cfg.n_nodes);
  return k;
}
void orkf_free(orkf* k) { delete k; }

// The kafka clients as ms_add_kafka_clients adds them: client i on server i mod n_nodes.  -2 where the engine refuses.
int orkf_add_clients(orkf* k, const orkf_config* kc, uint32_t first_name) {
  or_sim* s = k->s;
  if (!k->clients.empty() || !kc || kc->n_clients == 0 || kc->interval_ns <= 0 || kc->timeout_ns < 0 ||
      (uint64_t)kc->assign_permille + kc->crash_permille > 1000 || kc->n_clients % s->cfg.n_nodes) return -2;
  k->cfg = *kc;
  if (k->cfg.timeout_ns == 0) k->cfg.timeout_ns = 5000 * kTickNs;     // client.clj:18-20
  k->first = (uint32_t)s->eps.size();
  for (uint32_t i = 0; i < kc->n_clients; i++) {
    Endpoint ep;
    ep.name = "c" + std::to_string(first_name + i);
    ep.kind = OR_KIND_GEN_CLIENT;
    ep.gen.node = i % s->cfg.n_nodes;
    ep.gen.ordinal = i;
    s->eps.push_back(ep);
  }
  k->clients.resize(kc->n_clients);
  return (int)k->first;
}

int orkf_run(orkf* k, int64_t until_ns) {                               // or_run over the round above
  int64_t stall_now = k->s->now;
  uint64_t stall_round = k->s->round;
  while (k->s->now < until_ns) {
    if (!k->round() || k->stalled(stall_now, stall_round)) return -3;
  }
  return 0;
}

int orkf_recv(orkf* k, uint32_t e, int64_t timeout_ns, or_msg* out) {   // or_recv over the round above
  or_sim* s = k->s;
  if (e >= s->eps.size() || !s->eps[e].live) return -1;
  const int64_t give_up = s->now + timeout_ns;
  int64_t stall_now = s->now;
  uint64_t stall_round = s->round;
  for (;;) {
    if (k->stalled(stall_now, stall_round)) return -3;
    if (!s->eps[e].mailbox.empty()) {
      *out = s->eps[e].mailbox.front();
      s->eps[e].mailbox.pop_front();
      return 1;
    }
    if (s->now >= give_up) return 0;
    if (!k->round()) return -3;
  }
}

// the records since the last call, in (time, order) order as ms_kafka_history_drain hands them over; out = NULL:
// how many there are
size_t orkf_history(orkf* k, orkf_hist* out, size_t cap) {
  std::stable_sort(k->hist.begin() + (long)k->drained, k->hist.end(), [](const orkf_hist& a, const orkf_hist& b) {
    return a.time_ns != b.time_ns ? a.time_ns < b.time_ns : a.order < b.order;
  });
  if (!out) return k->hist.size() - k->drained;
  const size_t n = std::min(cap, k->hist.size() - k->drained);
  std::memcpy(out, k->hist.data() + k->drained, n * sizeof(orkf_hist));
  k->drained += n;
  return n;
}

// as ms_kafka_log: the log's length, and its first cap messages
size_t orkf_log(orkf* k, uint32_t node, uint32_t key, uint32_t* out, size_t cap) {
  if (node >= k->nodes.size()) return 0;
  auto it = k->nodes[node].queues.find(key);
  if (it == k->nodes[node].queues.end()) return 0;
  if (out) std::memcpy(out, it->second.data(), std::min(cap, it->second.size()) * 4);
  return it->second.size();
}

int64_t orkf_committed(orkf* k, uint32_t node, uint32_t key) {
  if (node >= k->nodes.size()) return -2;
  auto it = k->nodes[node].committed.find(key);
  return it == k->nodes[node].committed.end() ? -1 : (int64_t)it->second;
}

}  // extern "C"
