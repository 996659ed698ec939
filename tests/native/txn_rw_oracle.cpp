// TEST INFRASTRUCTURE: the oracle twin of the txn-rw-register workload (MS_W_TXN_RW, DESIGN.md 2.17), written apart
// from the device code (csrc/ms_raft.cuh rw_task / rw_handle, csrc/ms_kernels.cu rw_gen_step).
//
// It is the CPU oracle (oracle/oracle.cpp, compiled into this unit as it is) plus the node of
// demo/clojure/txn_rw_register_hat.clj on node.clj and the client of workload/txn_rw_register.clj:108-136 driven by the
// generator of the engine's header (ms_add_txn_rw_clients).  The node follows the Clojure closely: a state of lamport
// and kv, an insertion-ordered map timestamp -> txn+ {txn, node set} of unreplicated txns, apply-txn+ with its
// timestamp comparison, replicate-step! over the first entry, and the replicate / replicate_ack handlers as node.clj
// hands them their bodies: a replicate's txn+s are string-keyed maps, so :ts and :txn look up nil, and the acks carry
// nil timestamps.  The device reduces all this to a log and a count; parity checks that reduction.  The round loop
// restates or_sim::run_round for what a txn-rw-register simulation contains: the injector, the nodes, host-visible
// clients, client sinks and the txn clients.  Send, queues, partitions, the journal and time are the oracle's.
//
//     g++ -O2 -std=c++17 -fPIC -shared tests/native/txn_rw_oracle.cpp -o tests/native/_build/libtxn_rw_oracle.so
#include <map>
#include <optional>
#include <set>

#include "../../oracle/oracle.cpp"

extern "C" {
typedef struct orrw_config {          // the engine's ms_txn_rw_gen_config, restated
  uint32_t n_clients, min_len, max_len, key_count;
  int64_t  interval_ns, timeout_ns, time_limit_ns, key_period_ns;
} orrw_config;
typedef struct orrw_hist {            // the engine's ms_txn_rw_hist, restated
  int64_t  time_ns;
  uint64_t order;
  uint32_t client, op;
  uint8_t  type, f;
  uint16_t error;
  uint32_t node, index, base;
  uint64_t ops;
  uint32_t reads[4];
} orrw_hist;
typedef struct orrw_entry {           // the engine's ms_txn_rw_entry, restated
  uint64_t lamport, ops;
  uint32_t base, reads[4], pad;
} orrw_entry;
}

namespace {
enum { T_TXN = 60, T_TXN_OK = 61, T_REPLICATE = 90, T_REPLICATE_ACK = 91 };
enum { HF_TXN_RW = 15 };
enum { H_INVOKE = 0, H_OK = 1, H_FAIL = 2, H_INFO = 3 };
constexpr uint32_t kNone = 0xFFFFFFFFu;

struct Ts {                                          // [lamport node-id] (:16-20)
  uint64_t lamport;
  uint32_t node;
  bool operator==(const Ts& o) const { return lamport == o.lamport && node == o.node; }
  int compare(const Ts& o) const {                   // Clojure's compare on vectors of equal length
    if (lamport != o.lamport) return lamport < o.lamport ? -1 : 1;
    return node == o.node ? 0 : (node < o.node ? -1 : 1);
  }
};
struct Mop { bool write; uint32_t key, value; };     // [f k v]; a read's v is 0 = nil until it is applied
struct TxnPlus {                                     // {:ts :txn :nodes}
  std::optional<Ts> ts;
  std::vector<Mop> txn;
  std::set<uint32_t> nodes;
};
// A txn+ of a replicate body as node.clj:178 parses it: a map with the string keys "ts", "txn", "nodes".  Looking it
// up by the keywords :ts, :txn and :nodes finds nothing.
struct StringKeyedTxnPlus {
  std::optional<Ts> kw_ts() const { return std::nullopt; }
  std::vector<Mop> kw_txn() const { return {}; }
  std::set<uint32_t> kw_nodes() const { return {}; }
};
struct Versioned { Ts ts; uint32_t value; };

struct RwNode {
  std::optional<uint32_t> node_id;                   // the promise of node.clj: delivered by the first init
  uint64_t lamport = 0;                              // state (:22-27)
  std::map<uint32_t, Versioned> kv;
  std::vector<std::pair<Ts, TxnPlus>> unreplicated;  // unreplicated-txns, in insertion order (:29-32)
  std::vector<orrw_entry> served;                    // the completed txns, as ms_txn_rw_log returns them
  int64_t wake = 0;                                  // the replication thread's next wake-up
};
}  // namespace

struct orrw {
  or_sim* s;
  uint32_t group, n_keys, log_cap;
  std::vector<RwNode> nodes;
  orrw_config cfg{};
  std::vector<orrw_hist> hist;
  size_t drained = 0;

  uint32_t block_of(uint32_t e) const { return e / group * group; }
  std::vector<uint32_t> other_node_ids(uint32_t e) const {       // node-ids minus self, in block order
    std::vector<uint32_t> v;
    for (uint32_t n = block_of(e); n < block_of(e) + group; n++) if (n != e) v.push_back(n);
    return v;
  }
  static or_msg msg(uint32_t src, uint32_t dest, uint16_t type, uint32_t p0) {
    or_msg m; std::memset(&m, 0, sizeof m);
    m.src = src; m.dest = dest; m.type = type; m.p0 = p0;
    return m;
  }

  // apply-txn+ (:34-71): assigns a timestamp when the txn+ has none, applies the mops in order
  TxnPlus apply_txn_plus(uint32_t e, std::optional<Ts> ts, std::vector<Mop> txn) {
    RwNode& nd = nodes[e];
    Ts t;
    if (ts) { t = *ts; nd.lamport = std::max(nd.lamport, ts->lamport + 1); }
    else { t = Ts{nd.lamport, *nd.node_id}; nd.lamport += 1; }
    for (Mop& m : txn) {
      auto it = nd.kv.find(m.key);
      if (!m.write) m.value = it == nd.kv.end() ? 0 : it->second.value;
      else if (!(it != nd.kv.end() && it->second.ts.compare(t) > 0)) nd.kv[m.key] = Versioned{t, m.value};
    }
    TxnPlus r;
    r.ts = t; r.txn = txn;
    return r;
  }

  // replicate-step! (:90-102), every period of the thread, before the node's receives
  void task(uint32_t e, std::vector<Emit>& out) {
    RwNode& nd = nodes[e];
    const int64_t period = (int64_t)s->cfg.gset_interval_ms * kTickNs;
    while (s->now >= nd.wake) {
      nd.wake += period;
      if (nd.unreplicated.empty()) continue;
      const uint32_t node = *nd.unreplicated.front().second.nodes.begin();   // (first (:nodes txn+))
      uint32_t n = 0;
      for (const auto& kv : nd.unreplicated) n += kv.second.nodes.count(node);
      out.push_back(Emit(msg(e, node, T_REPLICATE, n)));
    }
  }

  void node(uint32_t e, const or_msg& m, std::vector<Emit>& out) {
    if (m.flags & OR_F_REPLY) return;                                    // handle-reply!: no rpcs
    RwNode& nd = nodes[e];
    if (m.type != OR_T_INIT && !nd.node_id) return;                      // waits on the node-id promise
    or_msg a; std::memset(&a, 0, sizeof a);
    a.src = e; a.dest = m.src;
    if (m.flags & OR_F_MSG_ID) { a.flags = OR_F_REPLY; a.in_reply_to = m.msg_id; }   // reply!: in_reply_to nil otherwise
    if (m.type == OR_T_INIT) {
      if (!nd.node_id) nd.node_id = e;                                   // deliver on a realized promise: no-op
      a.type = OR_T_INIT_OK;
    } else if (m.type == T_TXN) {                                        // (:116-125)
      std::vector<Mop> txn;
      uint32_t slot[4];
      for (int i = 0; i < 4; i++) {
        const uint32_t op = (uint32_t)(m.p1 >> (16 * i)) & 0xFFFF;
        if (!(op & 0x8000)) continue;
        if ((op & 0x3FFF) >= n_keys) { s->error = "txn-rw oracle: key out of range"; return; }
        slot[txn.size()] = i;
        txn.push_back(Mop{(op & 0x4000) != 0, op & 0x3FFF, m.p0 + (uint32_t)i});
      }
      if (nd.served.size() >= log_cap) { s->error = "txn-rw oracle: log full"; return; }
      TxnPlus t = apply_txn_plus(e, std::nullopt, txn);
      t.nodes.clear();                                                   // later-replicate!
      for (uint32_t n : other_node_ids(e)) t.nodes.insert(n);
      nd.unreplicated.emplace_back(*t.ts, t);
      orrw_entry en; std::memset(&en, 0, sizeof en);
      en.lamport = t.ts->lamport; en.ops = m.p1; en.base = m.p0;
      for (size_t j = 0; j < t.txn.size(); j++) if (!t.txn[j].write) en.reads[slot[j]] = t.txn[j].value;
      a.type = T_TXN_OK;
      a.p0 = (uint32_t)nd.served.size();
      a.p1 = t.ts->lamport;
      nd.served.push_back(en);
    } else if (m.type == T_REPLICATE) {                                  // (:127-145)
      const std::vector<StringKeyedTxnPlus> txns(m.p0);
      std::vector<std::optional<Ts>> tss;
      for (const StringKeyedTxnPlus& tp : txns) {
        apply_txn_plus(e, tp.kw_ts(), tp.kw_txn());
        std::set<uint32_t> nodes_ = tp.kw_nodes();
        nodes_.erase(e);
        if (!nodes_.empty()) { s->error = "txn-rw oracle: a replicated txn+ named nodes"; return; }
        tss.push_back(tp.kw_ts());
      }
      for (uint32_t n : other_node_ids(e)) out.push_back(Emit(msg(e, n, T_REPLICATE_ACK, (uint32_t)tss.size())));
      return;
    } else if (m.type == T_REPLICATE_ACK) {                              // (:147-166): every ts in :tss is nil
      for (uint32_t k = 0; k < m.p0; k++) {
        const std::optional<Ts> ts;
        for (auto& kv : nd.unreplicated)
          if (ts && kv.first == *ts) kv.second.nodes.erase(m.src);        // (get uts nil): never found
      }
      return;
    } else {
      a.type = OR_T_ERROR;                                               // "Unknown request type", {:code 10}
      a.p0 = 10;
    }
    out.push_back(Emit(a));
  }

  void record(uint32_t e, uint8_t type, uint16_t err, uint32_t index, const uint32_t reads[4]) {
    const Endpoint::Gen& g = s->eps[e].gen;
    orrw_hist h; std::memset(&h, 0, sizeof h);
    h.time_ns = s->now; h.order = (s->round << 24) | g.ordinal; h.client = e; h.op = g.ops;
    h.type = type; h.f = HF_TXN_RW; h.error = err;
    h.node = g.node; h.index = index; h.base = g.cur_value; h.ops = ops_of[g.ordinal];
    for (int i = 0; i < 4; i++) h.reads[i] = reads ? reads[i] : 0;
    hist.push_back(h);
  }
  std::vector<uint64_t> ops_of;                                          // the micro-ops of each client's txn in flight

  // a reply delivered to client e: only the awaited id counts (client.clj:106-107); with-errors #{}
  void reply(uint32_t e, const or_msg& m) {
    Endpoint::Gen& g = s->eps[e].gen;
    if (!(m.flags & OR_F_REPLY) || g.waiting_for == 0 || m.in_reply_to != g.waiting_for) return;
    g.waiting_for = 0;
    if (m.type == OR_T_ERROR) {
      record(e, m.p0 == 0 || m.p0 == 13 ? H_INFO : H_FAIL, (uint16_t)m.p0, kNone, nullptr);
      return;
    }
    const std::vector<orrw_entry>& log = nodes[g.node].served;
    if (m.p0 >= log.size()) { s->error = "txn-rw oracle: txn_ok names no logged txn"; return; }
    record(e, H_OK, 0, m.p0, log[m.p0].reads);
  }

  // after the replies of the round: the timeout, then at most one invocation
  void step(uint32_t e, std::vector<Emit>& out) {
    Endpoint::Gen& g = s->eps[e].gen;
    const int64_t now = s->now;
    if (g.waiting_for && now >= g.deadline_ns) {
      record(e, H_INFO, 0xFFFF, kNone, nullptr);
      g.waiting_for = 0;
    }
    if (g.waiting_for || g.phase != 0) return;
    if (now >= cfg.time_limit_ns) { g.phase = 3; return; }
    if (now < g.next_op_ns) return;
    const uint32_t key[2] = {s->cfg.seed_lo, s->cfg.seed_hi};
    const uint32_t c0[4] = {g.ops, e, 0xC11E47u, 0u}, c1[4] = {g.ops, e, 0xC11E47u, 1u};
    uint32_t x[4], y[4];
    philox(c0, key, x);
    philox(c1, key, y);
    const uint64_t base = 1 + 4 * ((uint64_t)g.ordinal + (uint64_t)cfg.n_clients * g.ops);
    if (base + 3 > 0xFFFFFFFFull) { s->error = "txn-rw oracle: value out of range"; return; }
    const uint32_t len = cfg.min_len + (uint32_t)(((uint64_t)x[0] * (cfg.max_len - cfg.min_len + 1)) >> 32);
    const uint64_t period = (uint64_t)(now / cfg.key_period_ns);
    uint64_t ops = 0;
    for (uint32_t i = 0; i < len; i++) {
      const uint64_t k = ((period % n_keys) * cfg.key_count + (((uint64_t)y[i] * cfg.key_count) >> 32)) % n_keys;
      const uint64_t w = (x[3] >> i) & 1;
      ops |= (0x8000 | w << 14 | k) << (16 * i);
    }
    g.next_op_ns = now + (int64_t)(((unsigned __int128)x[1] * (unsigned __int128)(2 * (uint64_t)cfg.interval_ns)) >> 32);
    g.ops++;
    g.cur_value = (uint32_t)base;
    ops_of[g.ordinal] = ops;
    g.waiting_for = ++g.next_msg_id;
    g.deadline_ns = now + cfg.timeout_ns;
    record(e, H_INVOKE, 0, kNone, nullptr);
    or_msg m = msg(e, g.node, T_TXN, (uint32_t)base);
    m.flags = OR_F_MSG_ID; m.msg_id = g.waiting_for; m.p1 = ops;
    out.push_back(Emit(m));
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
      if (ep.kind == OR_KIND_SERVER) task(e, out);
      while (!ep.q.empty() && ep.q.top().m.deadline_ns <= o.now) {
        const or_msg m = ep.q.top().m;
        ep.q.pop();
        if (o.partitioned(m.src, e)) continue;
        o.log_event(true, m);
        switch (ep.kind) {
          case OR_KIND_CLIENT: case OR_KIND_HOST: ep.mailbox.push_back(m); break;
          case OR_KIND_SIM_CLIENT: if (m.flags & OR_F_REPLY) o.client_replies++; break;
          case OR_KIND_GEN_CLIENT: reply(e, m); break;
          case OR_KIND_SERVER: node(e, m, out); break;
          default: o.error = "txn-rw oracle: no services here"; return false;
        }
        if (!o.error.empty()) return false;
      }
      if (ep.kind == OR_KIND_GEN_CLIENT) step(e, out);
      if (!o.error.empty()) return false;
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

// The txn-rw-register nodes of a fresh oracle made with workload 10: blocks of the oracle's raft_group servers (0 = all),
// n_keys keys (0 = 1024) and logs of log_cap txns (0 = 4096); the replication thread sleeps gset_interval_ms.
orrw* orrw_new(or_sim* s, uint32_t n_keys, uint32_t log_cap) {
  orrw* r = new orrw();
  r->s = s;
  r->group = s->cfg.raft_group ? s->cfg.raft_group : s->cfg.n_nodes;
  r->n_keys = n_keys ? n_keys : 1024;
  r->log_cap = log_cap ? log_cap : 4096;
  r->nodes.resize(s->cfg.n_nodes);
  for (RwNode& nd : r->nodes) nd.wake = (int64_t)s->cfg.gset_interval_ms * kTickNs;   // (Thread/sleep 100) first
  return r;
}
void orrw_free(orrw* r) { delete r; }

// The clients as ms_add_txn_rw_clients adds them: client i on server i mod n_nodes.  -2 where the engine refuses.
int orrw_add_clients(orrw* r, const orrw_config* rc, uint32_t first_name) {
  or_sim* s = r->s;
  if (r->cfg.n_clients || !rc || rc->n_clients == 0 || rc->interval_ns <= 0 || rc->timeout_ns < 0 || rc->key_period_ns <= 0 ||
      rc->min_len < 1 || rc->min_len > rc->max_len || rc->max_len > 4 || rc->key_count == 0 || rc->key_count > r->n_keys ||
      rc->n_clients % s->cfg.n_nodes) return -2;
  r->cfg = *rc;
  if (r->cfg.timeout_ns == 0) r->cfg.timeout_ns = 5000 * kTickNs;       // client.clj:18-20
  const uint32_t first = (uint32_t)s->eps.size();
  for (uint32_t i = 0; i < rc->n_clients; i++) {
    Endpoint ep;
    ep.name = "c" + std::to_string(first_name + i);
    ep.kind = OR_KIND_GEN_CLIENT;
    ep.gen.node = i % s->cfg.n_nodes;
    ep.gen.ordinal = i;
    s->eps.push_back(ep);
  }
  r->ops_of.assign(rc->n_clients, 0);
  return (int)first;
}

int orrw_run(orrw* r, int64_t until_ns) {                               // or_run over the round above
  int64_t stall_now = r->s->now;
  uint64_t stall_round = r->s->round;
  while (r->s->now < until_ns) {
    if (!r->round() || r->stalled(stall_now, stall_round)) return -3;
  }
  return 0;
}

int orrw_recv(orrw* r, uint32_t e, int64_t timeout_ns, or_msg* out) {   // or_recv over the round above
  or_sim* s = r->s;
  if (e >= s->eps.size() || !s->eps[e].live) return -1;
  const int64_t give_up = s->now + timeout_ns;
  int64_t stall_now = s->now;
  uint64_t stall_round = s->round;
  for (;;) {
    if (r->stalled(stall_now, stall_round)) return -3;
    if (!s->eps[e].mailbox.empty()) {
      *out = s->eps[e].mailbox.front();
      s->eps[e].mailbox.pop_front();
      return 1;
    }
    if (s->now >= give_up) return 0;
    if (!r->round()) return -3;
  }
}

// the records since the last call, in (time, order) order as ms_txn_rw_history_drain hands them over; out = NULL:
// how many there are
size_t orrw_history(orrw* r, orrw_hist* out, size_t cap) {
  std::stable_sort(r->hist.begin() + (long)r->drained, r->hist.end(), [](const orrw_hist& a, const orrw_hist& b) {
    return a.time_ns != b.time_ns ? a.time_ns < b.time_ns : a.order < b.order;
  });
  if (!out) return r->hist.size() - r->drained;
  const size_t n = std::min(cap, r->hist.size() - r->drained);
  std::memcpy(out, r->hist.data() + r->drained, n * sizeof(orrw_hist));
  r->drained += n;
  return n;
}

// as ms_txn_rw_log: the log's length, and its first cap entries
size_t orrw_log(orrw* r, uint32_t node, orrw_entry* out, size_t cap) {
  if (node >= r->nodes.size()) return 0;
  const std::vector<orrw_entry>& log = r->nodes[node].served;
  if (out) std::memcpy(out, log.data(), std::min(cap, log.size()) * sizeof(orrw_entry));
  return log.size();
}

// as ms_txn_rw_state; also the size of the unreplicated map and the smallest pending node set's size
int orrw_state(orrw* r, uint32_t node, uint64_t* lamport, uint32_t* log_len, uint32_t* value, uint64_t* ts, size_t cap,
               uint32_t* unreplicated, uint32_t* min_pending) {
  if (node >= r->nodes.size()) return -2;
  const RwNode& nd = r->nodes[node];
  *lamport = nd.lamport;
  *log_len = (uint32_t)nd.served.size();
  for (size_t k = 0; k < cap && k < r->n_keys; k++) {
    auto it = nd.kv.find((uint32_t)k);
    value[k] = it == nd.kv.end() ? 0 : it->second.value;
    ts[k] = it == nd.kv.end() ? 0 : it->second.ts.lamport;
  }
  *unreplicated = (uint32_t)nd.unreplicated.size();
  uint32_t mn = kNone;
  for (const auto& kv : nd.unreplicated) mn = std::min<uint32_t>(mn, (uint32_t)kv.second.nodes.size());
  *min_pending = mn;
  return (int)r->n_keys;
}

}  // extern "C"
