// TEST INFRASTRUCTURE: the oracle twin of the lin-kv proxy (MS_W_KV_PROXY, DESIGN.md 2.14), written apart from the
// device code (csrc/ms_raft.cuh kp_handle).
//
// It is the kv-oracle twin (tests/native/kv_oracle.cpp, which is the CPU oracle plus the closed-loop lin-kv clients,
// both compiled into this unit as they are) plus the proxy node of demo/ruby/lin_kv_proxy.rb on node.rb.  The round
// loop below restates or_sim::run_round for what a proxy simulation contains: the injector, the proxies, the kv
// services they forward to, host-visible clients, client sinks and the lin-kv clients.  Send, queues, the services'
// state machines, the clients, the journal and time are the oracle's and the twin's own code.
//
//     g++ -O2 -std=c++17 -fPIC -shared tests/native/kv_proxy_oracle.cpp -o tests/native/_build/libkv_proxy_oracle.so
#include "kv_oracle.cpp"

namespace {
struct ProxyNode {             // LinKVNode (lin_kv_proxy.rb) on Node (node.rb)
  struct Closure { uint32_t client = 0, client_msg_id = 0; bool had_msg_id = false; };
  bool crashed = false;                                          // main! raised: the process is gone
  uint32_t next_msg_id = 0;                                      // @next_msg_id (node.rb:10)
  std::map<uint32_t, Closure> callbacks;                         // @callbacks by msg_id: the newest cb_slots ids only
};
const char* const kServiceNames[3] = {"lin-kv", "seq-kv", "lww-kv"};
}  // namespace

struct orkp {
  or_sim* s;
  uint32_t service;                   // OR_SVC_LIN_KV / _SEQ_KV / _LWW_KV
  std::vector<ProxyNode> nodes;       // by server index
  orkv* kv = nullptr;                 // the lin-kv clients, once added

  // main! (node.rb:153-169) takes a message with in_reply_to to its callback (none: ignored), anything else to the
  // handler of its type; proxy! (lin_kv_proxy.rb:27-38) rpc!s the request body minus msg_id to the service, and its
  // callback reply!s the service's body minus msg_id.  No handler: main! raises and the node process is dead.
  void node(uint32_t e, const or_msg& m, std::vector<Emit>& out) {
    ProxyNode& pn = nodes[e];
    if (pn.crashed) return;
    auto answer = [&](uint32_t client, uint32_t client_msg_id, bool had_msg_id, uint16_t type, uint16_t flags,
                      uint32_t p0, uint64_t p1) {                                // reply! (node.rb:88-91)
      or_msg a; std::memset(&a, 0, sizeof a);
      a.src = e; a.dest = client; a.type = type; a.p0 = p0; a.p1 = p1;
      a.flags = flags & ~(OR_F_MSG_ID | OR_F_REPLY);
      if (had_msg_id) { a.flags |= OR_F_REPLY; a.in_reply_to = client_msg_id; }   // else "in_reply_to": null
      out.push_back(Emit(a));
    };
    if (m.flags & OR_F_REPLY) {
      auto it = pn.callbacks.find(m.in_reply_to);
      if (it == pn.callbacks.end()) return;                                      // "Ignoring reply ... with no callback"
      const ProxyNode::Closure cb = it->second;
      pn.callbacks.erase(it);
      answer(cb.client, cb.client_msg_id, cb.had_msg_id, m.type, m.flags, m.p0, m.p1);
      return;
    }
    if (m.type == OR_T_INIT) { answer(m.src, m.msg_id, (m.flags & OR_F_MSG_ID) != 0, OR_T_INIT_OK, 0, 0, 0); return; }
    if (m.type == OR_T_READ || m.type == OR_T_WRITE || m.type == OR_T_CAS) {
      int svc = -1;
      for (uint32_t i = s->cfg.n_nodes; i < s->eps.size(); i++)
        if (s->eps[i].live && s->eps[i].kind == OR_KIND_SERVICE && s->eps[i].name == kServiceNames[service]) svc = (int)i;
      if (svc < 0) { s->error = std::string("Invalid dest for message: ") + kServiceNames[service]; return; }
      const uint32_t id = ++pn.next_msg_id;                                      // rpc! (node.rb:95-102)
      pn.callbacks.erase(id - s->cb_slots);                                     // the table keeps the newest ids only
      pn.callbacks[id] = ProxyNode::Closure{m.src, m.msg_id, (m.flags & OR_F_MSG_ID) != 0};
      or_msg q; std::memset(&q, 0, sizeof q);
      q.src = e; q.dest = (uint32_t)svc; q.type = m.type; q.p0 = m.p0; q.p1 = m.p1;
      q.flags = OR_F_MSG_ID | (m.flags & OR_F_CREATE); q.msg_id = id;
      out.push_back(Emit(q));
      return;
    }
    pn.crashed = true;                                                          // raise "No handler for ..."
  }

  // service-thread (service.clj:245-263) as or_sim::run_round runs it: rand-int is word 3 of the Philox draw of the
  // emission the reply would be
  void service_step(uint32_t e, const or_msg& m, std::vector<Emit>& out) {
    or_body q;
    q.type = m.type; q.flags = m.flags; q.msg_id = m.msg_id; q.in_reply_to = m.in_reply_to; q.p0 = m.p0; q.p1 = m.p1;
    const uint32_t ctr[4] = {(uint32_t)out.size(), e, (uint32_t)s->round, (uint32_t)(s->round >> 32)};
    const uint32_t key[2] = {s->cfg.seed_lo, s->cfg.seed_hi};
    uint32_t x[4];
    philox(ctr, key, x);
    const SvcReply r = s->eps[e].svc.handle(m.src, q, x[3]);
    if (!r.reply) return;
    or_msg rm = or_sim::reply_to(m, r.type);
    rm.p0 = r.p0; rm.p1 = r.p1;
    out.push_back(Emit(rm));
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
      if (ep.kind == OR_KIND_GEN_CLIENT && !kv) { o.error = "kv proxy oracle: lin-kv clients not added here"; return false; }
      out.clear();
      while (!ep.q.empty() && ep.q.top().m.deadline_ns <= o.now) {
        const or_msg m = ep.q.top().m;
        ep.q.pop();
        if (o.partitioned(m.src, e)) continue;
        o.log_event(true, m);
        switch (ep.kind) {
          case OR_KIND_CLIENT: case OR_KIND_HOST: ep.mailbox.push_back(m); break;
          case OR_KIND_SIM_CLIENT: if (m.flags & OR_F_REPLY) o.client_replies++; break;
          case OR_KIND_GEN_CLIENT: kv->reply(e, m); break;
          case OR_KIND_SERVICE: service_step(e, m, out); break;
          default: node(e, m, out);
        }
        if (!o.error.empty()) return false;
      }
      if (ep.kind == OR_KIND_GEN_CLIENT) kv->step(e, out);
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

// The proxies of a fresh oracle made with workload 6 and n_nodes servers; NULL for a service that is not a kv store.
orkp* orkp_new(or_sim* s, uint32_t service) {
  if (service > OR_SVC_LWW_KV) return nullptr;
  orkp* k = new orkp();
  k->s = s;
  k->service = service;
  k->nodes.resize(s->cfg.n_nodes);
  return k;
}
void orkp_free(orkp* k) {
  delete k->kv;
  delete k;
}

// The lin-kv clients as ms_add_kv_clients adds them to MS_W_KV_PROXY: kv_oracle.cpp's binding, roles and generator,
// with one key range per group (the proxies share one store, the service's).  NULL where the engine refuses.
int orkp_add_clients(orkp* k, const orkv_config* kc, uint32_t first_name) {
  or_sim* s = k->s;
  if (k->kv || !kc || kc->n_clients == 0 || kc->interval_ns <= 0 || kc->keys_per_group == 0 || kc->key_period_ns <= 0 ||
      kc->value_range > 256) return -2;
  const uint32_t g = s->cfg.raft_group ? s->cfg.raft_group : s->cfg.n_nodes;
  const uint32_t clusters = s->cfg.n_nodes / g;
  if (kc->n_clients % (2 * g)) return -2;
  orkv* kv = new orkv();
  kv->s = s;
  kv->cfg = *kc;
  if (kv->cfg.value_range == 0) kv->cfg.value_range = 5;                  // (rand-int 5)
  if (kv->cfg.timeout_ns <= 0)                                            // lin_kv.clj:54
    kv->cfg.timeout_ns = (int64_t)std::max<uint64_t>(10ull * s->cfg.latency_mean_ms, 1000ull) * kTickNs;
  kv->first = (uint32_t)s->eps.size();
  for (uint32_t i = 0; i < kc->n_clients; i++) {
    const uint32_t group = i / (2 * g);
    Endpoint ep;
    ep.name = "c" + std::to_string(first_name + i);
    ep.kind = OR_KIND_GEN_CLIENT;
    ep.gen.node = (group % clusters) * g + i % g;
    ep.gen.ordinal = i;
    s->eps.push_back(ep);
    kv->clients.push_back(KvClient{group * kc->keys_per_group, i % (2 * g) < g});
  }
  k->kv = kv;
  return (int)kv->first;
}

int orkp_run(orkp* k, int64_t until_ns) {                                 // or_run over the round above
  int64_t stall_now = k->s->now;
  uint64_t stall_round = k->s->round;
  while (k->s->now < until_ns) {
    if (!k->round() || k->stalled(stall_now, stall_round)) return -3;
  }
  return 0;
}

int orkp_recv(orkp* k, uint32_t e, int64_t timeout_ns, or_msg* out) {     // or_recv over the round above
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

// out = {crashed, the last msg_id sent, closures pending, 0, 0, 0, 0, 0}, as ms_raft_state on MS_W_KV_PROXY
int orkp_state(orkp* k, uint32_t node, uint64_t out[8]) {
  if (node >= k->nodes.size()) return -1;
  const ProxyNode& pn = k->nodes[node];
  out[0] = pn.crashed; out[1] = pn.next_msg_id; out[2] = pn.callbacks.size();
  for (int i = 3; i < 8; i++) out[i] = 0;
  return 0;
}

}  // extern "C"
