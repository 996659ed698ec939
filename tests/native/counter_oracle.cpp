// TEST INFRASTRUCTURE: the oracle twin of the g-counter and pn-counter workloads (MS_W_G_COUNTER / MS_W_PN_COUNTER,
// DESIGN.md 2.16), written apart from the device code (csrc/ms_raft.cuh ct_task / ct_handle, csrc/ms_kernels.cu
// ct_gen_step).
//
// It is the CPU oracle (oracle/oracle.cpp, compiled into this unit as it is) plus the PN-counter node of
// demo/ruby/pn_counter.rb on crdt.rb and node.rb, and the client of workload/pn_counter.clj:35-53 driven by the
// generator of the engine's header (ms_add_gen_clients).  The node keeps two maps node id -> count, merged key-wise by
// max, as the Ruby does; a merge's value is the sender's maps as they were at the run that sent it.  The round loop
// below restates or_sim::run_round for what a counter simulation contains: the injector, the nodes, host-visible
// clients, client sinks and the counter clients.  Send, queues, partitions, the journal, the history and time are the
// oracle's.
//
//     g++ -O2 -std=c++17 -fPIC -shared tests/native/counter_oracle.cpp -o tests/native/_build/libcounter_oracle.so
#include <map>

#include "../../oracle/oracle.cpp"

extern "C" {
typedef struct orct_config {          // the engine's ms_gen_config, restated
  uint32_t n_clients, read_permille;
  int64_t  interval_ns, timeout_ns, time_limit_ns, quiet_ns;
} orct_config;
}

namespace {
enum { T_MERGE = 80, T_MERGE_OK = 81 };
enum { W_G_COUNTER = 8, W_PN_COUNTER = 9 };
enum { HF_READ = 1, HF_ADD = 14 };
enum { H_INVOKE = 0, H_OK = 1, H_INFO = 3 };
enum { MIX = 0, QUIET = 1, FINAL = 2, DONE = 3 };

struct Counter {                                     // PNCounter: a GCounter of increments and one of decrements
  std::map<uint32_t, int64_t> inc, dec;              // node_id => value_at_node (pn_counter.rb:10-13)
  int64_t read() const {
    int64_t v = 0;
    for (const auto& kv : inc) v += kv.second;
    for (const auto& kv : dec) v -= kv.second;
    return v;
  }
  void merge(const Counter& o) {                     // @counters.merge(other) { [v1, v2].max }
    for (const auto& kv : o.inc) inc[kv.first] = std::max(inc[kv.first], kv.second);
    for (const auto& kv : o.dec) dec[kv.first] = std::max(dec[kv.first], kv.second);
  }
};

struct CounterNode {
  Counter value;
  bool crashed = false;                              // main! raised: the process is gone
  bool running = false;                              // the `every 5` task was started by an init
  int64_t next_run = 0;
  uint32_t runs = 0;
};
}  // namespace

struct orct {
  or_sim* s;
  uint32_t group;                                    // servers per block (node_ids of an init)
  std::vector<CounterNode> nodes;
  std::map<std::pair<uint32_t, uint32_t>, Counter> sent;   // (sender, run) -> the value its merges carry
  orct_config cfg{};

  uint32_t block_of(uint32_t e) const { return e / group * group; }
  uint32_t block_end(uint32_t e) const { return std::min<uint32_t>(block_of(e) + group, s->cfg.n_nodes); }

  // `every 5` of crdt.rb:41-45: other_node_ids in order, each sent the value
  void task(uint32_t e, std::vector<Emit>& out) {
    CounterNode& nd = nodes[e];
    if (nd.crashed || !nd.running || s->now < nd.next_run) return;
    const uint32_t k = ++nd.runs;
    sent[std::make_pair(e, k)] = nd.value;
    for (uint32_t other = block_of(e); other < block_end(e); other++) {
      if (other == e) continue;
      or_msg m; std::memset(&m, 0, sizeof m);
      m.src = e; m.dest = other; m.type = T_MERGE; m.p1 = k;
      out.push_back(Emit(m));
    }
    nd.next_run += (int64_t)s->cfg.gset_interval_ms * kTickNs;
  }

  // main! (node.rb:149-185) and the handlers of crdt.rb / pn_counter.rb, one message at a time
  void node(uint32_t e, const or_msg& m, std::vector<Emit>& out) {
    CounterNode& nd = nodes[e];
    if (nd.crashed) return;
    if (m.flags & OR_F_REPLY) return;                                  // no callbacks: "Ignoring reply"
    if (m.type == T_MERGE_OK) return;
    or_msg a; std::memset(&a, 0, sizeof a);
    a.src = e; a.dest = m.src;
    if (m.flags & OR_F_MSG_ID) { a.flags = OR_F_REPLY; a.in_reply_to = m.msg_id; }   // reply!: in_reply_to nil otherwise
    if (m.type == OR_T_INIT) {
      nd.running = true;
      nd.next_run = s->now;                                            // start_periodic_tasks!: runs at once
      a.type = OR_T_INIT_OK;
    } else if (m.type == OR_T_ADD) {
      const int32_t delta = (int32_t)m.p0;
      if (delta >= 0) nd.value.inc[e] += delta;
      else nd.value.dec[e] += -(int64_t)delta;
      a.type = OR_T_ADD_OK;
    } else if (m.type == OR_T_READ) {
      a.type = OR_T_READ_OK;
      a.p1 = (uint64_t)nd.value.read();
    } else if (m.type == T_MERGE) {
      const auto it = sent.find(std::make_pair(m.src, (uint32_t)m.p1));
      if (m.src < block_of(e) || m.src >= block_end(e) || m.src == e || m.p1 >> 32 || it == sent.end()) {
        s->error = "counter oracle: merge of a value no block member's task sent";
        return;
      }
      nd.value.merge(it->second);
      a.type = T_MERGE_OK;
    } else {
      nd.crashed = true;                                               // "No handler for ...": the process exits
      return;
    }
    out.push_back(Emit(a));
  }

  // a reply delivered to client e: only the awaited id counts (client.clj:106-107); no with-errors
  void reply(uint32_t e, const or_msg& m) {
    Endpoint::Gen& g = s->eps[e].gen;
    if (!(m.flags & OR_F_REPLY) || g.waiting_for == 0 || m.in_reply_to != g.waiting_for) return;
    g.waiting_for = 0;
    if (m.type == OR_T_ERROR) { s->gen_hist(e, g.ops, H_INFO, (uint8_t)g.cur_f, (uint16_t)m.p0, g.cur_value); return; }
    uint32_t value = g.cur_value;
    if (g.cur_f == HF_READ) {
      const int64_t v = (int64_t)m.p1;
      if (v < INT32_MIN || v > INT32_MAX) { s->error = "counter oracle: read value out of int32"; return; }
      value = (uint32_t)(int32_t)v;
    }
    s->gen_hist(e, g.ops, H_OK, (uint8_t)g.cur_f, 0, value);
  }

  // after the replies of the round: the timeout, then at most one invocation
  void step(uint32_t e, std::vector<Emit>& out) {
    Endpoint::Gen& g = s->eps[e].gen;
    const int64_t now = s->now;
    if (g.waiting_for && now >= g.deadline_ns) {
      s->gen_hist(e, g.ops, H_INFO, (uint8_t)g.cur_f, 0xFFFF, g.cur_value);
      g.waiting_for = 0;
    }
    if (g.waiting_for) return;
    bool invoke = false;
    uint32_t f = HF_READ, value = 0;
    if (g.phase == MIX) {
      if (now >= cfg.time_limit_ns) {
        g.phase = QUIET;
      } else if (now >= g.next_op_ns) {
        const uint32_t ctr[4] = {g.ops, e, 0xC11E47u, 0u};
        const uint32_t key[2] = {s->cfg.seed_lo, s->cfg.seed_hi};
        uint32_t x[4];
        philox(ctr, key, x);
        if ((((uint64_t)x[0] * 1000u) >> 32) >= cfg.read_permille) {
          f = HF_ADD;
          const int32_t delta = s->cfg.workload == W_PN_COUNTER ? (int32_t)(((uint64_t)x[2] * 10u) >> 32) - 5   // (- (rand-int 10) 5)
                                                                : (int32_t)(((uint64_t)x[2] * 5u) >> 32);
          value = (uint32_t)delta;
        }
        g.next_op_ns = now + (int64_t)(((unsigned __int128)x[1] * (unsigned __int128)(2 * (uint64_t)cfg.interval_ns)) >> 32);
        invoke = true;
      }
    }
    if (g.phase == QUIET && now >= cfg.time_limit_ns + cfg.quiet_ns) { g.phase = FINAL; invoke = true; }
    else if (g.phase == FINAL && !invoke) g.phase = DONE;
    if (!invoke) return;
    g.ops++;
    g.cur_f = f; g.cur_value = value;
    g.waiting_for = ++g.next_msg_id;
    g.deadline_ns = now + cfg.timeout_ns;
    s->gen_hist(e, g.ops, H_INVOKE, (uint8_t)f, 0, value);
    or_msg m; std::memset(&m, 0, sizeof m);
    m.src = e; m.dest = g.node; m.flags = OR_F_MSG_ID; m.msg_id = g.waiting_for;
    m.type = f == HF_READ ? OR_T_READ : OR_T_ADD;
    m.p0 = value;
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
          default: o.error = "counter oracle: no services here"; return false;
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

// The counter nodes of a fresh oracle made with workload 8 or 9: blocks of the oracle's raft_group servers (0 = all).
orct* orct_new(or_sim* s) {
  orct* c = new orct();
  c->s = s;
  c->group = s->cfg.raft_group ? s->cfg.raft_group : s->cfg.n_nodes;
  c->nodes.resize(s->cfg.n_nodes);
  return c;
}
void orct_free(orct* c) { delete c; }

// The clients as ms_add_gen_clients adds them: client i on server i mod n_nodes.  -2 where the engine refuses.
int orct_add_clients(orct* c, const orct_config* gc, uint32_t first_name) {
  or_sim* s = c->s;
  if (c->cfg.n_clients || !gc || gc->n_clients == 0 || gc->interval_ns <= 0 || gc->read_permille > 1000) return -2;
  c->cfg = *gc;
  if (c->cfg.timeout_ns <= 0) c->cfg.timeout_ns = 5000 * kTickNs;       // client.clj:18-20
  if (c->cfg.quiet_ns <= 0) c->cfg.quiet_ns = 10000 * kTickNs;          // core.clj:75-78
  const uint32_t first = (uint32_t)s->eps.size();
  for (uint32_t i = 0; i < gc->n_clients; i++) {
    Endpoint ep;
    ep.name = "c" + std::to_string(first_name + i);
    ep.kind = OR_KIND_GEN_CLIENT;
    ep.gen.node = i % s->cfg.n_nodes;
    ep.gen.ordinal = i;
    s->eps.push_back(ep);
  }
  return (int)first;
}

int orct_run(orct* c, int64_t until_ns) {                               // or_run over the round above
  int64_t stall_now = c->s->now;
  uint64_t stall_round = c->s->round;
  while (c->s->now < until_ns) {
    if (!c->round() || c->stalled(stall_now, stall_round)) return -3;
  }
  return 0;
}

int orct_recv(orct* c, uint32_t e, int64_t timeout_ns, or_msg* out) {   // or_recv over the round above
  or_sim* s = c->s;
  if (e >= s->eps.size() || !s->eps[e].live) return -1;
  const int64_t give_up = s->now + timeout_ns;
  int64_t stall_now = s->now;
  uint64_t stall_round = s->round;
  for (;;) {
    if (c->stalled(stall_now, stall_round)) return -3;
    if (!s->eps[e].mailbox.empty()) {
      *out = s->eps[e].mailbox.front();
      s->eps[e].mailbox.pop_front();
      return 1;
    }
    if (s->now >= give_up) return 0;
    if (!c->round()) return -3;
  }
}

// as ms_counter_state: inc then dec of node's block members, in block order; returns the count
int orct_state(orct* c, uint32_t node, int64_t* out, size_t cap) {
  if (node >= c->nodes.size()) return -2;
  const Counter& v = c->nodes[node].value;
  const uint32_t lo = c->block_of(node), n = c->block_end(node) - lo;
  for (uint32_t i = 0; i < 2 * n && i < cap; i++) {
    const std::map<uint32_t, int64_t>& m = i < n ? v.inc : v.dec;
    const auto it = m.find(lo + i % n);
    out[i] = it == m.end() ? 0 : it->second;
  }
  return (int)(2 * n);
}

}  // extern "C"
