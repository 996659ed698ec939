// TEST INFRASTRUCTURE: the oracle twin of the engine's closed-loop lin-kv clients (ms_add_kv_clients,
// DESIGN.md 2.12), written apart from the device code (csrc/ms_kernels.cu kv_gen_step).
//
// It is the CPU oracle (oracle/oracle.cpp, compiled into this unit as it is) plus the worker of
// workload/lin_kv.clj:40-85 as one more endpoint program.  A client's request leaves in the client's place in
// the round, in endpoint order, so the round loop below restates or_sim::run_round for what a Raft lin-kv
// simulation contains: the injector, Raft servers, client sinks and these clients.  Everything else about a
// round (send, queues, the Raft node, the journal, time) is the oracle's own code.
//
//     g++ -O2 -std=c++17 -fPIC -shared tests/native/kv_oracle.cpp -o tests/native/_build/libkv_oracle.so
#include "../../oracle/oracle.cpp"

extern "C" {
typedef struct orkv_config {          // the engine's ms_kv_gen_config, restated
  uint32_t n_clients, value_range, keys_per_group;
  int64_t  interval_ns, timeout_ns, time_limit_ns, key_period_ns;
} orkv_config;
}

namespace {
enum { HF_KV_READ = 2, HF_KV_WRITE = 3, HF_KV_CAS = 4 };   // or_hist.f; value = key | a << 16 | b << 24

struct KvClient { uint32_t key_base; bool reader; };
}  // namespace

struct orkv {
  or_sim* s;
  orkv_config cfg;
  uint32_t first;                     // endpoint index of client 0
  std::vector<KvClient> clients;      // by ordinal

  // a reply delivered to client e: the leader answers a proxied request, not the node asked
  // (raft.py:558-561), so the id alone decides
  void reply(uint32_t e, const or_msg& m) {
    Endpoint::Gen& g = s->eps[e].gen;
    if (!(m.flags & OR_F_REPLY) || g.waiting_for == 0 || m.in_reply_to != g.waiting_for) return;
    const bool read = g.cur_f == HF_KV_READ;
    if (m.type == OR_T_ERROR) {
      const bool indefinite = m.p0 == 0 || m.p0 == 13;                  // errors.edn
      s->gen_hist(e, g.ops, (read || !indefinite) ? 2 : 3, (uint8_t)g.cur_f, (uint16_t)m.p0, g.cur_value);   // lin_kv.clj:52
    } else {
      s->gen_hist(e, g.ops, 1, (uint8_t)g.cur_f, 0, read ? g.cur_value | (uint32_t)((m.p1 & 0xFF) << 16) : g.cur_value);
    }
    g.waiting_for = 0;
  }

  // after the replies of the round: the timeout, then at most one invocation
  void step(uint32_t e, std::vector<Emit>& out) {
    Endpoint::Gen& g = s->eps[e].gen;
    const KvClient& c = clients[g.ordinal];
    const int64_t now = s->now;
    if (g.waiting_for) {
      if (now < g.deadline_ns) return;
      s->gen_hist(e, g.ops, g.cur_f == HF_KV_READ ? 2 : 3, (uint8_t)g.cur_f, 0xFFFF, g.cur_value);
      g.waiting_for = 0;
    }
    if (g.phase != 0) return;
    if (now >= cfg.time_limit_ns) { g.phase = 3; return; }              // no quiet period, no final read
    if (now < g.next_op_ns) return;
    const uint32_t ctr[4] = {g.ops, e, 0xC11E47u, 0u};
    const uint32_t key[2] = {s->cfg.seed_lo, s->cfg.seed_hi};
    uint32_t x[4];
    philox(ctr, key, x);
    or_msg m; std::memset(&m, 0, sizeof m);
    const uint32_t k = c.key_base + (uint32_t)(((uint64_t)now / (uint64_t)cfg.key_period_ns) % cfg.keys_per_group);
    const uint32_t v0 = (uint32_t)(((uint64_t)x[2] * cfg.value_range) >> 32);
    const uint32_t v1 = (uint32_t)(((uint64_t)x[3] * cfg.value_range) >> 32);
    uint32_t hv = k;
    if (c.reader) { g.cur_f = HF_KV_READ; m.type = OR_T_READ; }
    else if ((((uint64_t)x[0] * 3u) >> 32) == 0) { g.cur_f = HF_KV_WRITE; m.type = OR_T_WRITE; m.p1 = v0; hv |= v0 << 16; }
    else { g.cur_f = HF_KV_CAS; m.type = OR_T_CAS; m.p1 = (uint64_t)v0 | ((uint64_t)v1 << 32); hv |= (v0 << 16) | (v1 << 24); }
    g.next_op_ns = now + (int64_t)(((unsigned __int128)x[1] * (unsigned __int128)(2 * (uint64_t)cfg.interval_ns)) >> 32);
    g.ops++;
    g.cur_value = hv;
    g.waiting_for = ++g.next_msg_id;
    g.deadline_ns = now + cfg.timeout_ns;
    s->gen_hist(e, g.ops, 0, (uint8_t)g.cur_f, 0, hv);
    m.src = e; m.dest = g.node; m.flags = OR_F_MSG_ID; m.msg_id = g.waiting_for; m.p0 = k;
    out.push_back(Emit(m));
  }

  // One round of a Raft lin-kv simulation with these clients: or_sim::run_round's four steps (injector,
  // endpoints in index order, visibility, time) with the client program in the endpoint step.
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
      if (ep.kind != OR_KIND_SERVER && ep.kind != OR_KIND_SIM_CLIENT && ep.kind != OR_KIND_GEN_CLIENT) {
        o.error = "kv oracle: only Raft servers, client sinks and the lin-kv clients";
        return false;
      }
      out.clear();
      if (ep.kind == OR_KIND_SERVER) ep.rn.draws = 0;
      while (!ep.q.empty() && ep.q.top().m.deadline_ns <= o.now) {
        const or_msg m = ep.q.top().m;
        ep.q.pop();
        if (o.partitioned(m.src, e)) continue;
        o.log_event(true, m);
        if (ep.kind == OR_KIND_SERVER) o.node_raft(e, m, out);
        else if (ep.kind == OR_KIND_GEN_CLIENT) reply(e, m);
        else if (m.flags & OR_F_REPLY) o.client_replies++;
        if (!o.error.empty()) return false;
      }
      if (ep.kind == OR_KIND_SERVER) o.raft_actions(e, out);
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
};

extern "C" {

// Adds the clients to a fresh or running OR_W_RAFT oracle; NULL on a configuration the engine refuses too.
orkv* orkv_add_clients(or_sim* s, const orkv_config* kc, uint32_t first_name) {
  if (!kc || kc->n_clients == 0 || kc->interval_ns <= 0 || kc->keys_per_group == 0 || kc->key_period_ns <= 0 ||
      kc->value_range > 256 || s->cfg.workload != OR_W_RAFT || s->gcfg.n_clients) return nullptr;
  const uint32_t g = s->cfg.raft_group ? s->cfg.raft_group : s->cfg.n_nodes;
  const uint32_t clusters = s->cfg.n_nodes / g;
  if (kc->n_clients % (2 * g)) return nullptr;
  orkv* k = new orkv();
  k->s = s;
  k->cfg = *kc;
  if (k->cfg.value_range == 0) k->cfg.value_range = 5;                    // (rand-int 5)
  if (k->cfg.timeout_ns <= 0)                                             // lin_kv.clj:54
    k->cfg.timeout_ns = (int64_t)std::max<uint64_t>(10ull * s->cfg.latency_mean_ms, 1000ull) * kTickNs;
  k->first = (uint32_t)s->eps.size();
  for (uint32_t i = 0; i < kc->n_clients; i++) {
    const uint32_t group = i / (2 * g);
    Endpoint ep;
    ep.name = "c" + std::to_string(first_name + i);
    ep.kind = OR_KIND_GEN_CLIENT;
    ep.gen.node = (group % clusters) * g + i % g;
    ep.gen.ordinal = i;
    s->eps.push_back(ep);
    k->clients.push_back(KvClient{(group / clusters) * kc->keys_per_group, i % (2 * g) < g});
  }
  return k;
}
void orkv_free(orkv* k) { delete k; }
uint32_t orkv_first(orkv* k) { return k->first; }

int orkv_run(orkv* k, int64_t until_ns) {                                 // or_run over the round above
  or_sim* s = k->s;
  int64_t stall_now = s->now;
  uint64_t stall_round = s->round;
  while (s->now < until_ns) {
    if (!k->round()) return -3;
    if (s->now != stall_now) { stall_now = s->now; stall_round = s->round; }
    else if (s->round - stall_round > (1ull << 20)) { s->error = "virtual time is not advancing"; return -3; }
  }
  return 0;
}

}  // extern "C"
