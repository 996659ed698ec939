// ms_raft.cuh -- the Raft node program of the lin-kv workload (SURVEY.md section 8a row N4),
// following demo/python/raft.py, the reference's single-threaded poll-loop node.  A node's step
// in a round is inherently sequential (one handler at a time, raft.py:577-584), so it is run by
// one thread of the node's CTA: every due message in id order through process_msg and the
// handlers, then one pass of the loop's actions in its own priority order.  What the step
// sends is staged in the node's row of `rf_stage`; the CTA then emits the staged records in
// parallel through the common path (Philox loss / latency, journal, ring scatter).
//
// Included by ms_kernels.cu inside namespace msd, after Rec / latch_error.
#pragma once

struct RaftCtx {
  const Params& p;
  DevState* st;
  uint32_t e;          // this node
  int64_t now;
  uint64_t round;
  RaftDev* r;
  uint4* log;          // this node's log (entry i, 1-based, at log[2 * (i - 1)])
  uint4* cb;           // this node's callback table
  uint4* stage;
  uint32_t n_stage;
  uint32_t draws;
  // the node's Raft cluster = node_ids of its init (raft.py:447-459): servers [gbase, gbase + gn).
  // One cluster of all servers by default; ms_config.reserved[4] = g runs independent clusters of g
  // consecutive servers (the leader tables and vote bitmaps are per cluster member).
  uint32_t gbase, gn;
};

__device__ __forceinline__ void rf_group_of(const Params& p, uint32_t e, uint32_t& gbase, uint32_t& gn) {
  const uint32_t G = p.rf_group ? p.rf_group : p.n_servers;
  gbase = (e / G) * G;
  gn = min(G, p.n_servers - gbase);
}

struct RaftEntry {     // {'term': t, 'op': body + 'client'}  (raft.py:118-121,553-556)
  uint32_t term, tf, key, client;
  uint64_t p1;
  uint32_t msg_id;
};

__device__ __forceinline__ RaftEntry rf_entry_unpack(uint4 a, uint4 b) {
  RaftEntry en;
  en.term = a.x; en.tf = a.y; en.key = a.z; en.client = a.w;
  en.p1 = (uint64_t)b.x | ((uint64_t)b.y << 32);
  en.msg_id = b.z;
  return en;
}
__device__ __forceinline__ void rf_entry_store(uint4* at, const RaftEntry& en) {
  at[0] = make_uint4(en.term, en.tf, en.key, en.client);
  at[1] = make_uint4((uint32_t)en.p1, (uint32_t)(en.p1 >> 32), en.msg_id, 0u);
}
__device__ __forceinline__ uint32_t rf_log_term(const RaftCtx& c, uint32_t index /* 1-based */) {
  return c.log[2 * (size_t)(index - 1)].x;
}

__device__ __forceinline__ void rf_emit(RaftCtx& c, const Rec& r) {
  if (c.n_stage >= c.p.rf_stage_cap) { latch_error(c.st, E_RAFT_CAPACITY, c.e); return; }
  uint4* at = c.stage + (size_t)c.n_stage * 3;
  at[0] = make_uint4(r.src, r.dest, r.msg_id, r.in_reply_to);
  at[1] = make_uint4(r.tf, r.p0, (uint32_t)r.p1, (uint32_t)(r.p1 >> 32));
  c.n_stage++;
}

// net.reply (raft.py:72-75): body + in_reply_to, back to the sender; no msg_id
__device__ __forceinline__ Rec rf_reply_to(const RaftCtx& c, const Rec& req, uint32_t type) {
  Rec r;
  r.round = 0; r.ticket = 0; r.idx = 0;
  r.src = c.e; r.dest = req.src; r.msg_id = 0; r.in_reply_to = req.msg_id;
  r.tf = type | ((uint32_t)MS_F_REPLY << 16);
  r.p0 = 0; r.p1 = 0;
  return r;
}

// random.random() (raft.py:251): word 0 of Philox(0x80000000 | k, node, round), k-th draw of this step
__device__ __forceinline__ uint32_t rf_draw(RaftCtx& c) {
  uint32_t x[4];
  philox4x32_10(0x80000000u | c.draws++, c.e, (uint32_t)c.round, (uint32_t)(c.round >> 32), c.p.seed_lo,
                c.p.seed_hi, x);
  return x[0];
}
__device__ __forceinline__ void rf_reset_election_deadline(RaftCtx& c) {          // raft.py:249-251
  const uint32_t x = rf_draw(c);
  c.r->election_deadline = c.now + kElectionTimeoutNs + (int64_t)(((uint64_t)x * (uint64_t)kElectionTimeoutNs) >> 32);
}
__device__ __forceinline__ void rf_reset_step_down_deadline(RaftCtx& c) {         // :253-255
  c.r->step_down_deadline = c.now + kElectionTimeoutNs;
}
__device__ __forceinline__ void rf_become_follower(RaftCtx& c) {                  // :307-314
  c.r->state = RAFT_FOLLOWER;
  c.r->leader = -1;
  rf_reset_election_deadline(c);
}
__device__ __forceinline__ void rf_maybe_step_down(RaftCtx& c, uint32_t remote_term) {   // :257-270
  if (c.r->term < remote_term) {
    c.r->term = remote_term;
    c.r->voted_for = -1;
    rf_become_follower(c);
  }
}

// net.rpc (raft.py:77-82): fresh msg_id, remember the closure, send
__device__ __forceinline__ void rf_rpc(RaftCtx& c, uint32_t dest, uint32_t type, uint32_t p0, uint64_t p1,
                                       uint32_t kind, uint32_t cb_node, int32_t cb_ni, uint32_t cb_n) {
  const uint32_t id = c.r->next_msg_id++;
  uint4* slot = c.cb + 2 * (size_t)(id & c.p.rf_cb_mask);
  slot[0] = make_uint4(id, kind, c.r->term, cb_node);
  slot[1] = make_uint4((uint32_t)cb_ni, cb_n, 0u, 0u);
  Rec r;
  r.round = 0; r.ticket = 0; r.idx = 0;
  r.src = c.e; r.dest = dest; r.msg_id = id; r.in_reply_to = 0;
  r.tf = type | ((uint32_t)MS_F_MSG_ID << 16);
  r.p0 = p0; r.p1 = p1;
  rf_emit(c, r);
}

__device__ void rf_become_candidate(RaftCtx& c) {                                 // :316-325 + request_votes :272-303
  RaftDev* r = c.r;
  r->state = RAFT_CANDIDATE;
  r->term += 1;
  r->voted_for = (int32_t)c.e;
  r->leader = -1;
  rf_reset_election_deadline(c);
  rf_reset_step_down_deadline(c);
  uint32_t* votes = c.p.rf_votes + (size_t)c.e * c.p.rf_vote_words;
  for (uint32_t w = 0; w < c.p.rf_vote_words; w++) votes[w] = 0;
  votes[(c.e - c.gbase) >> 5] |= 1u << ((c.e - c.gbase) & 31);
  r->n_votes = 1;
  const uint64_t last = (uint64_t)r->log_size | ((uint64_t)rf_log_term(c, r->log_size) << 32);
  for (uint32_t n = c.gbase; n < c.gbase + c.gn; n++)                             // brpc, :243-246
    if (n != c.e) rf_rpc(c, n, MS_T_REQUEST_VOTE, r->term, last, 1u, 0u, 0, 0u);
}

__device__ void rf_become_leader(RaftCtx& c) {                                    // :327-339
  RaftDev* r = c.r;
  r->state = RAFT_LEADER;
  r->leader = -1;
  r->last_replication = 0;
  int32_t* next = c.p.rf_next + (size_t)c.e * c.p.rf_gmax;
  int32_t* match = c.p.rf_match + (size_t)c.e * c.p.rf_gmax;
  for (uint32_t n = 0; n < c.gn; n++) { next[n] = (int32_t)r->log_size + 1; match[n] = 0; }
  rf_reset_step_down_deadline(c);
}

// process_msg + handlers (raft.py:84-111, 443-573).  `return` where the reference raises: the
// main loop catches, the message is consumed and nothing else happens (raft.py:585-588).
__device__ void rf_handle(RaftCtx& c, const Rec& m) {
  RaftDev* r = c.r;
  const uint32_t type = m.tf & 0xFFFFu, flags = m.tf >> 16;
  if (flags & MS_F_REPLY) {                                                       // :97-101
    uint4* slot = c.cb + 2 * (size_t)(m.in_reply_to & c.p.rf_cb_mask);
    const uint4 s0 = slot[0], s1 = slot[1];
    if (s0.y == 0 || s0.x != m.in_reply_to) return;                               // KeyError
    slot[0] = make_uint4(0u, 0u, 0u, 0u);                                         // del self.callbacks[m]
    const uint32_t cb_term = s0.z, cb_node = s0.w;
    if (s0.y == 1) {                                                              // request_votes' handle, :282-303
      rf_reset_step_down_deadline(c);
      rf_maybe_step_down(c, m.p0);
      if (r->state == RAFT_CANDIDATE && r->term == cb_term && m.p0 == r->term && m.p1 != 0 &&
          m.src >= c.gbase && m.src < c.gbase + c.gn) {
        uint32_t* votes = c.p.rf_votes + (size_t)c.e * c.p.rf_vote_words;
        const uint32_t v = m.src - c.gbase, bit = 1u << (v & 31);
        if (!(votes[v >> 5] & bit)) { votes[v >> 5] |= bit; r->n_votes++; }
        if (c.gn / 2 + 1 <= r->n_votes) rf_become_leader(c);
      }
    } else {                                                                      // replicate_log's handler, :413-426
      rf_maybe_step_down(c, m.p0);
      if (r->state == RAFT_LEADER && cb_term == r->term) {
        rf_reset_step_down_deadline(c);
        int32_t* next = c.p.rf_next + (size_t)c.e * c.p.rf_gmax;
        int32_t* match = c.p.rf_match + (size_t)c.e * c.p.rf_gmax;
        const int32_t ni = (int32_t)s1.x, ne = (int32_t)s1.y;
        const uint32_t cn = cb_node - c.gbase;                                  // member index of the closure's node
        if (cn < c.gn) {
          if (m.p1 != 0) {
            if (next[cn] < ni + ne) next[cn] = ni + ne;
            if (match[cn] < ni - 1 + ne) match[cn] = ni - 1 + ne;
          } else {
            next[cn] -= 1;
          }
        }
      }
    }
    return;
  }
  if (type == MS_T_INIT) {                                                        // :447-459
    if (r->state != RAFT_NASCENT) return;                                         // "Can't init twice!"
    rf_become_follower(c);
    rf_emit(c, rf_reply_to(c, m, MS_T_INIT_OK));
    return;
  }
  if (type == MS_T_REQUEST_VOTE) {                                                // :464-495
    rf_maybe_step_down(c, m.p0);
    bool grant = false;
    const uint32_t last_log_index = (uint32_t)m.p1, last_log_term = (uint32_t)(m.p1 >> 32);
    const uint32_t my_last_term = rf_log_term(c, r->log_size);
    if (m.p0 < r->term) {
    } else if (r->voted_for >= 0) {
    } else if (last_log_term < my_last_term) {
    } else if (last_log_term == my_last_term && last_log_index < r->log_size) {
    } else {
      grant = true;
      r->voted_for = (int32_t)m.src;
      rf_reset_election_deadline(c);
    }
    Rec res = rf_reply_to(c, m, MS_T_REQUEST_VOTE_RES);
    res.p0 = r->term; res.p1 = grant ? 1u : 0u;
    rf_emit(c, res);
    return;
  }
  if (type == MS_T_APPEND_ENTRIES) {                                              // :499-545
    rf_maybe_step_down(c, m.p0);
    Rec res = rf_reply_to(c, m, MS_T_APPEND_ENTRIES_RES);
    res.p0 = r->term; res.p1 = 0;
    if (m.p0 < r->term) { rf_emit(c, res); return; }
    r->leader = (int32_t)m.src;
    rf_reset_election_deadline(c);
    // the payload: the sender's k-th append_entries, in the payload heap
    const uint32_t k = (uint32_t)m.p1;
    if (m.src >= c.p.n_servers) return;
    // the payload lives in the heap of the sender's shard (NVLink peer memory when that is not ours)
    const uint32_t o = owner_of(m.src, c.p.n_servers, c.p.n_shards);
    const uint4* heap = c.p.rf_heap_sh[o];
    if (__ldcg(c.p.rf_ext_tag_sh[o] + (size_t)m.src * kRaftExt + k % kRaftExt) != k) return;             // forged handle
    const uint64_t off = __ldcg(c.p.rf_ext_off_sh[o] + (size_t)m.src * kRaftExt + k % kRaftExt);
    const uint4 guard = __ldcg(heap + (off & c.p.rf_heap_mask));
    if (guard.x != m.src || guard.y != k) { latch_error(c.st, E_SNAPSHOT, m.src); return; }               // overwritten
    const uint4 hd = __ldcg(heap + ((off + 1) & c.p.rf_heap_mask));
    const uint32_t prev_log_index = hd.x, prev_log_term = hd.y, leader_commit = hd.z, n_entries = hd.w;
    if (prev_log_index == 0) return;                                              // "Out of bounds previous log index"
    if (prev_log_index > r->log_size || rf_log_term(c, prev_log_index) != prev_log_term) {
      rf_emit(c, res);                                                            // we disagree on the previous term
      return;
    }
    if (prev_log_index + n_entries > c.p.rf_log_cap) { latch_error(c.st, E_RAFT_CAPACITY, c.e); return; }
    for (uint32_t q = 0; q < n_entries; q++) {                                    // truncate + append, :533-534
      c.log[2 * (size_t)(prev_log_index + q)] = __ldcg(heap + ((off + 2 + 2 * (uint64_t)q) & c.p.rf_heap_mask));
      c.log[2 * (size_t)(prev_log_index + q) + 1] = __ldcg(heap + ((off + 3 + 2 * (uint64_t)q) & c.p.rf_heap_mask));
    }
    r->log_size = prev_log_index + n_entries;
    if (r->commit_index < leader_commit) r->commit_index = leader_commit < r->log_size ? leader_commit : r->log_size;
    res.p1 = 1;
    rf_emit(c, res);
    return;
  }
  if (type == MS_T_READ || type == MS_T_WRITE || type == MS_T_CAS) {              // kv_req, :550-570
    if (r->state == RAFT_LEADER) {
      if (m.p0 >= c.p.rf_n_keys) { latch_error(c.st, E_VALUE_RANGE, m.p0); return; }
      if (r->log_size >= c.p.rf_log_cap) { latch_error(c.st, E_RAFT_CAPACITY, c.e); return; }
      RaftEntry en;
      en.term = r->term; en.tf = m.tf; en.key = m.p0; en.client = m.src; en.p1 = m.p1; en.msg_id = m.msg_id;
      rf_entry_store(c.log + 2 * (size_t)r->log_size, en);
      r->log_size++;
    } else if (r->leader >= 0) {
      Rec f = m;                                                                  // msg['dest'] = leader; send_msg(msg)
      f.dest = (uint32_t)r->leader;
      rf_emit(c, f);
    } else {
      Rec res = rf_reply_to(c, m, MS_T_ERROR);
      res.p0 = 11;                                                                // not a leader
      rf_emit(c, res);
    }
    return;
  }
  // 'No callback or handler': RuntimeError, message consumed
}

// KVStore.apply (raft.py:158-192)
__device__ Rec rf_apply(RaftCtx& c, const RaftEntry& op) {
  Rec res;
  res.round = 0; res.ticket = 0; res.idx = 0;
  res.src = c.e; res.dest = op.client; res.msg_id = 0; res.in_reply_to = op.msg_id;
  res.p0 = 0; res.p1 = 0;
  uint32_t otype = MS_T_ERROR;
  uint32_t* val = c.p.rf_kv_val + (size_t)c.e * c.p.rf_n_keys + op.key;
  uint8_t* has = c.p.rf_kv_has + (size_t)c.e * c.p.rf_n_keys + op.key;
  const uint32_t type = op.tf & 0xFFFFu;
  if (type == MS_T_READ) {
    if (*has) { otype = MS_T_READ_OK; res.p1 = *val; } else res.p0 = 20;
  } else if (type == MS_T_WRITE) {
    if (!*has) c.r->kv_size++;
    *val = (uint32_t)op.p1; *has = 1;
    otype = MS_T_WRITE_OK;
  } else {
    if (!*has) res.p0 = 20;
    else if (*val != (uint32_t)op.p1) res.p0 = 22;
    else { *val = (uint32_t)(op.p1 >> 32); otype = MS_T_CAS_OK; }
  }
  res.tf = otype | ((uint32_t)MS_F_REPLY << 16);
  return res;
}

// One pass of the main loop's actions once the inbox is empty (raft.py:577-584), in the loop's
// priority order; time is frozen inside a round, so each is idle again right after it ran.
__device__ void rf_actions(RaftCtx& c) {
  RaftDev* r = c.r;
  const uint32_t N = c.gn;                                                                // cluster size
  if (r->state == RAFT_LEADER && r->step_down_deadline < c.now) rf_become_follower(c);   // :371-376
  {                                                                                       // replicate_log, :387-441
    const int64_t elapsed = c.now - r->last_replication;
    bool replicated = false, aborted = false;
    const uint32_t first_rpc = r->next_msg_id;          // RPCs of this pass: ids first_rpc .. next_msg_id - 1
    uint32_t last_node = 0, last_n = 0;
    int32_t last_ni = 0;
    if (r->state == RAFT_LEADER && kMinReplicationNs < elapsed) {
      const int32_t* next = c.p.rf_next + (size_t)c.e * c.p.rf_gmax;
      for (uint32_t n = c.gbase; n < c.gbase + N; n++) {
        if (n == c.e) continue;
        const int32_t ni = next[n - c.gbase];
        if (ni <= 0) { aborted = true; break; }                                           // from_index raises (:147-148): the
                                                                                          // iteration ends, later ones raise again
        const int32_t n_entries = (int32_t)r->log_size - ni + 1 > 0 ? (int32_t)r->log_size - ni + 1 : 0;
        if (0 < n_entries || kHeartbeatNs < elapsed) {
          // log.get(ni - 1) = entries[ni - 2]; Python's entries[-1] when ni == 1 is the last entry
          const int32_t pi = ni - 2;
          if (pi >= (int32_t)r->log_size) { aborted = true; break; }                      // IndexError
          const uint32_t prev_term = pi < 0 ? rf_log_term(c, r->log_size) : rf_log_term(c, (uint32_t)pi + 1);
          const uint32_t k = ++r->appends;
          const uint64_t words = 2 + 2 * (uint64_t)n_entries;
          if (words > c.p.rf_heap_mask) { latch_error(c.st, E_RAFT_CAPACITY, c.e); aborted = true; break; }
          const uint64_t off = atomicAdd(c.p.rf_heap_cursor, (unsigned long long)words);
          c.p.rf_heap[off & c.p.rf_heap_mask] = make_uint4(c.e, k, 0u, 0u);
          c.p.rf_heap[(off + 1) & c.p.rf_heap_mask] = make_uint4((uint32_t)(ni - 1), prev_term, r->commit_index, (uint32_t)n_entries);
          for (int32_t q = 0; q < n_entries; q++) {
            c.p.rf_heap[(off + 2 + 2 * (uint64_t)q) & c.p.rf_heap_mask] = c.log[2 * (size_t)(ni - 1 + q)];
            c.p.rf_heap[(off + 3 + 2 * (uint64_t)q) & c.p.rf_heap_mask] = c.log[2 * (size_t)(ni - 1 + q) + 1];
          }
          c.p.rf_ext_off[(size_t)c.e * kRaftExt + k % kRaftExt] = off;
          c.p.rf_ext_tag[(size_t)c.e * kRaftExt + k % kRaftExt] = k;
          rf_rpc(c, n, MS_T_APPEND_ENTRIES, r->term, k, 2u, n, ni, (uint32_t)n_entries);
          last_node = n; last_ni = ni; last_n = (uint32_t)n_entries;
          replicated = true;
        }
      }
    }
    // Python closures bind late: `handler` reads _ni / _entries / _node (raft.py:408-426) from the
    // frame of this replicate_log call when the reply arrives, i.e. the values of the LAST node the
    // pass sent to, for every RPC of the pass (pinned by tests/test_raft_reference.py)
    for (uint32_t id = first_rpc; id != r->next_msg_id; id++) {
      uint4* slot = c.cb + 2 * (size_t)(id & c.p.rf_cb_mask);
      if (slot[0].y == 2u && slot[0].x == id) {
        slot[0].w = last_node;
        slot[1] = make_uint4((uint32_t)last_ni, last_n, 0u, 0u);
      }
    }
    if (aborted) return;
    if (replicated) r->last_replication = c.now;
  }
  if (r->election_deadline < c.now) {                                                     // election, :358-367
    if (r->state == RAFT_FOLLOWER || r->state == RAFT_CANDIDATE) rf_become_candidate(c);
    else rf_reset_election_deadline(c);
  }
  if (r->state == RAFT_LEADER) {                                                          // advance_commit_index, :378-385
    int32_t* xs = c.p.rf_scratch + (size_t)c.e * c.p.rf_gmax;
    const int32_t* match = c.p.rf_match + (size_t)c.e * c.p.rf_gmax;
    for (uint32_t n = 0; n < N; n++) {                                                    // insertion sort of match_index()
      const int32_t v = n == c.e - c.gbase ? (int32_t)r->log_size : match[n];
      uint32_t j = n;
      while (j > 0 && xs[j - 1] > v) { xs[j] = xs[j - 1]; j--; }
      xs[j] = v;
    }
    const int32_t nmed = xs[N - (N / 2 + 1)];                                             // median, :29-33
    if ((int32_t)r->commit_index < nmed && rf_log_term(c, (uint32_t)nmed) == r->term) r->commit_index = (uint32_t)nmed;
  }
  while (r->last_applied < r->commit_index) {                                             // advance_state_machine, :343-354
    r->last_applied += 1;
    const RaftEntry op = rf_entry_unpack(c.log[2 * (size_t)(r->last_applied - 1)], c.log[2 * (size_t)(r->last_applied - 1) + 1]);
    const Rec res = rf_apply(c, op);
    if (r->state == RAFT_LEADER) rf_emit(c, res);
  }
}

// After a node's step: does replicate_log have a reason to run again before the heartbeat interval
// (a follower behind the log, or a next_index that makes it raise)?  k_snapshot uses it, with the
// node's deadlines, to skip the rounds in which the node's step would do nothing.
__device__ void rf_note_busy(RaftCtx& c) {
  RaftDev* r = c.r;
  uint32_t busy = 0;
  if (r->state == RAFT_LEADER) {
    const int32_t* next = c.p.rf_next + (size_t)c.e * c.p.rf_gmax;
    for (uint32_t n = 0; n < c.gn && !busy; n++)
      if (n != c.e - c.gbase && (next[n] <= 0 || next[n] <= (int32_t)r->log_size)) busy = 1;
  }
  r->busy = busy;
}

// k_snapshot: would this node's step do anything in a round at time `now` with an empty inbox?
// The conditions are the guards of rf_actions, verbatim (a skipped step must be a no-op).
__device__ __forceinline__ bool rf_timer_due(const RaftDev& r, int64_t now) {
  if (r.election_deadline < now) return true;                                             // election (also a nascent node's reset)
  if (r.state != RAFT_LEADER) return false;
  if (r.step_down_deadline < now) return true;
  const int64_t elapsed = now - r.last_replication;
  return kMinReplicationNs < elapsed && (r.busy || kHeartbeatNs < elapsed);
}
// The earliest instant at which rf_timer_due holds (k_wake, ms_set_idle_jump): its guards with their strict `<`.
// Keep the two in step.
__device__ __forceinline__ int64_t rf_wake_ns(const RaftDev& r) {
  auto after = [](int64_t t, int64_t d) { return t > INT64_MAX - d - 1 ? INT64_MAX : t + d + 1; };
  int64_t w = after(r.election_deadline, 0);
  if (r.state != RAFT_LEADER) return w;
  w = min(w, after(r.step_down_deadline, 0));
  return min(w, after(r.last_replication, r.busy ? kMinReplicationNs : kHeartbeatNs));
}

// ------------------------------------------------------------------ txn-list-append, single key
// demo/clojure/single_key_txn.clj: the whole database is one value under key "root" (key 0) of
// the lin-kv service (:134-141).  handle-txn! (:163-173) = read the root, apply-txn, cas the
// root from what was read to the result (create_if_not_exists), answer txn_ok -- or error 30
// when the cas fails with 22.  Database values travel as version ids (include/maelstrom_b200.h):
// apply-txn (:115-127) is a pure function of (value, txn), so the node only has to know whether
// the txn appends.  Every request runs in its own future (:93-95): the two RPCs of a txn are
// closures in the node's table, like Raft's.  Uses RaftDev.next_msg_id / .appends (versions minted).
__device__ void txn_handle(RaftCtx& c, const Rec& m) {
  RaftDev* r = c.r;
  const uint32_t type = m.tf & 0xFFFFu, flags = m.tf >> 16;
  const uint32_t lin_kv = c.p.sv_ep[MS_SVC_LIN_KV];
  if (flags & MS_F_REPLY) {                                                       // handle-reply!, :60-68
    uint4* slot = c.cb + 2 * (size_t)(m.in_reply_to & c.p.rf_cb_mask);
    const uint4 s0 = slot[0], s1 = slot[1];
    if (s0.y == 0 || s0.x != m.in_reply_to) return;                               // no such future
    slot[0] = make_uint4(0u, 0u, 0u, 0u);
    Rec req;                                                                      // the txn request being served
    req.round = 0; req.ticket = 0; req.idx = 0;
    req.src = s0.w; req.dest = c.e; req.msg_id = s0.z; req.in_reply_to = 0; req.tf = MS_T_TXN; req.p0 = 0; req.p1 = 0;
    if (s0.y == 3) {                                                              // read-service, :143-150
      uint32_t old_v;
      if (type == MS_T_READ_OK) old_v = (uint32_t)m.p1;
      else if (type == MS_T_ERROR && m.p0 == 20) old_v = 0;                       // not found: nil
      else { Rec er = rf_reply_to(c, req, MS_T_ERROR); er.p0 = m.p0; rf_emit(c, er); return; }   // :99-103
      uint32_t new_v;
      if (s1.y) new_v = 2u + c.e + c.p.n_servers * (r->appends++);               // an append: a value nobody has seen
      else new_v = old_v == 0 ? 1u : old_v;                                       // reads only: unchanged ({} for nil)
      const uint32_t id = ++r->next_msg_id;                                       // (swap! next-message-id inc), :54
      uint4* s2 = c.cb + 2 * (size_t)(id & c.p.rf_cb_mask);
      s2[0] = make_uint4(id, 4u, s0.z, s0.w);
      s2[1] = make_uint4(old_v, new_v, 0u, 0u);
      Rec q;                                                                      // cas-service!, :152-161
      q.round = 0; q.ticket = 0; q.idx = 0;
      q.src = c.e; q.dest = lin_kv; q.msg_id = id; q.in_reply_to = 0;
      q.tf = MS_T_CAS | ((uint32_t)(MS_F_MSG_ID | MS_F_CREATE) << 16);
      q.p0 = 0; q.p1 = (uint64_t)old_v | ((uint64_t)new_v << 32);
      rf_emit(c, q);
    } else if (s0.y == 4) {                                                       // :168-173
      if (type == MS_T_CAS_OK) {
        Rec ok = rf_reply_to(c, req, MS_T_TXN_OK);
        ok.p1 = (uint64_t)s1.x | ((uint64_t)s1.y << 32);
        rf_emit(c, ok);
      } else {
        Rec er = rf_reply_to(c, req, MS_T_ERROR);
        er.p0 = (type == MS_T_ERROR && m.p0 == 22) ? 30u : m.p0;                  // "root altered"
        rf_emit(c, er);
      }
    }
    return;
  }
  if (type == MS_T_INIT) { rf_emit(c, rf_reply_to(c, m, MS_T_INIT_OK)); return; }   // :70-77
  if (type == MS_T_TXN) {                                                         // handle-txn!, :163-173
    if (lin_kv == 0xFFFFFFFFu) { latch_error(c.st, E_INVALID_DEST, lin_kv); return; }   // no lin-kv service
    const uint32_t id = ++r->next_msg_id;
    uint4* s2 = c.cb + 2 * (size_t)(id & c.p.rf_cb_mask);
    s2[0] = make_uint4(id, 3u, m.msg_id, m.src);
    s2[1] = make_uint4(0u, (flags & MS_F_APPENDS) ? 1u : 0u, 0u, 0u);
    Rec q;
    q.round = 0; q.ticket = 0; q.idx = 0;
    q.src = c.e; q.dest = lin_kv; q.msg_id = id; q.in_reply_to = 0;
    q.tf = MS_T_READ | ((uint32_t)MS_F_MSG_ID << 16);
    q.p0 = 0; q.p1 = 0;
    rf_emit(c, q);
    return;
  }
  Rec er = rf_reply_to(c, m, MS_T_ERROR);                                         // "Unknown request type", :85-88
  er.p0 = 10;
  rf_emit(c, er);
}

// ------------------------------------------------------------------ lin-kv proxy
// demo/ruby/lin_kv_proxy.rb on node.rb (DESIGN.md 2.14): read / write / cas are forwarded to the backing service
// (Params.kp_service) by rpc!, and the service's reply, minus its msg_id, goes back to the client by reply!.  Handlers
// run in dequeue order, a legal schedule of Ruby's thread per message.  Uses RaftDev.state (1 = crashed: main! raised
// on a message without a handler), .next_msg_id (@next_msg_id) and .kv_size (closures pending).  A closure is
// {msg_id, 1, the client's msg_id, the client} + {the request had a msg_id}.
__device__ void kp_answer(RaftCtx& c, uint32_t client, uint32_t client_msg_id, bool had_msg_id, uint32_t type,
                          uint32_t flags, uint32_t p0, uint64_t p1) {
  Rec a;                                                                          // reply! (node.rb:88-91)
  a.round = 0; a.ticket = 0; a.idx = 0;
  a.src = c.e; a.dest = client; a.msg_id = 0;
  a.in_reply_to = had_msg_id ? client_msg_id : 0u;                                // in_reply_to: nil without a msg_id
  flags &= ~(uint32_t)(MS_F_MSG_ID | MS_F_REPLY);
  a.tf = type | ((flags | (had_msg_id ? (uint32_t)MS_F_REPLY : 0u)) << 16);
  a.p0 = p0; a.p1 = p1;
  rf_emit(c, a);
}

__device__ void kp_handle(RaftCtx& c, const Rec& m) {
  RaftDev* r = c.r;
  if (r->state) return;                                                           // crashed: read, never acted on
  const uint32_t type = m.tf & 0xFFFFu, flags = m.tf >> 16;
  if (flags & MS_F_REPLY) {                                                       // main!, node.rb:159-164
    uint4* slot = c.cb + 2 * (size_t)(m.in_reply_to & c.p.rf_cb_mask);
    const uint4 s0 = slot[0], s1 = slot[1];
    if (s0.y == 0 || s0.x != m.in_reply_to) return;                               // "Ignoring reply ... with no callback"
    slot[0] = make_uint4(0u, 0u, 0u, 0u);
    r->kv_size--;
    kp_answer(c, s0.w, s0.z, s1.x != 0, type, flags, m.p0, m.p1);                 // proxy!'s block
    return;
  }
  if (type == MS_T_INIT) {                                                        // node.rb:22-36
    kp_answer(c, m.src, m.msg_id, (flags & MS_F_MSG_ID) != 0, MS_T_INIT_OK, 0u, 0u, 0ull);
    return;
  }
  if (type == MS_T_READ || type == MS_T_WRITE || type == MS_T_CAS) {              // proxy!, lin_kv_proxy.rb:27-38
    const uint32_t svc = c.p.sv_ep[c.p.kp_service];
    if (svc == 0xFFFFFFFFu) { latch_error(c.st, E_INVALID_DEST, svc); return; }   // no such service endpoint
    const uint32_t id = ++r->next_msg_id;                                         // rpc!, node.rb:95-102
    uint4* slot = c.cb + 2 * (size_t)(id & c.p.rf_cb_mask);
    if (slot[0].y == 0) r->kv_size++;                                             // else it takes an older closure's slot
    slot[0] = make_uint4(id, 1u, m.msg_id, m.src);
    slot[1] = make_uint4((flags & MS_F_MSG_ID) ? 1u : 0u, 0u, 0u, 0u);
    Rec q;
    q.round = 0; q.ticket = 0; q.idx = 0;
    q.src = c.e; q.dest = svc; q.msg_id = id; q.in_reply_to = 0;
    q.tf = type | ((uint32_t)(MS_F_MSG_ID | (flags & MS_F_CREATE)) << 16);
    q.p0 = m.p0; q.p1 = m.p1;
    rf_emit(c, q);
    return;
  }
  r->state = 1;                                                                   // "No handler": main! raises, node.rb:167
}

// ------------------------------------------------------------------ kafka, single node
// demo/clojure/kafka_single_node.clj (DESIGN.md 2.15): every node keeps its own append-only log per key
// (Params.kf_log / kf_len) and committed offsets (kf_committed, kKafkaAbsent = none).  Handlers run in dequeue
// order, a legal schedule of the demo's future per message.  A poll_ok carries the log lengths, not the messages:
// the log never changes below its length, so ms_kafka_log gives them afterwards.  Keys of a request are checked
// before any effect; slot 0 is applied before slot 1.
__device__ __forceinline__ bool kf_keys_ok(RaftCtx& c, uint32_t keys) {
  for (int i = 0; i < 2; i++) {
    const uint32_t k = (keys >> (16 * i)) & 0xFFFFu;
    if (k != kKafkaNoKey && k >= c.p.kf_keys) { latch_error(c.st, E_VALUE_RANGE, k); return false; }
  }
  return true;
}

__device__ void kf_handle(RaftCtx& c, const Rec& m) {
  const uint32_t type = m.tf & 0xFFFFu, flags = m.tf >> 16;
  if (flags & MS_F_REPLY) return;                                                 // handle-reply!: no rpcs of its own (:80-88)
  const bool has_id = (flags & MS_F_MSG_ID) != 0;
  Rec a;                                                                          // reply! (:65-68)
  a.round = 0; a.ticket = 0; a.idx = 0;
  a.src = c.e; a.dest = m.src; a.msg_id = 0;
  a.in_reply_to = has_id ? m.msg_id : 0u;                                         // in_reply_to: nil without a msg_id
  a.p0 = 0; a.p1 = 0;
  const size_t row = (size_t)c.e * c.p.kf_keys;
  uint32_t* len = c.p.kf_len + row;
  uint32_t* committed = c.p.kf_committed + row;
  uint32_t out_type = MS_T_ERROR;
  if (type == MS_T_INIT) {                                                        // handle-init! (:90-97)
    out_type = MS_T_INIT_OK;
  } else if (type == MS_T_SEND) {                                                 // handle-send! (:197-207)
    const uint32_t k = m.p0;
    if (k >= c.p.kf_keys) { latch_error(c.st, E_VALUE_RANGE, k); return; }
    const uint32_t n = len[k];
    if (n >= c.p.kf_cap) { latch_error(c.st, E_KAFKA_CAPACITY, c.e); return; }
    c.p.kf_log[(row + k) * c.p.kf_cap + n] = (uint32_t)m.p1;
    len[k] = n + 1u;
    out_type = MS_T_SEND_OK;
    a.p1 = n;                                                                     // (dec (count queue'))
  } else if (type == MS_T_POLL) {                                                 // handle-poll! (:174-195)
    if (!kf_keys_ok(c, m.p0)) return;
    uint32_t keys = 0xFFFFFFFFu;
    for (int i = 0; i < 2; i++) {
      const uint32_t k = (m.p0 >> (16 * i)) & 0xFFFFu, o = (uint32_t)(m.p1 >> (32 * i));
      if (k == kKafkaNoKey || o >= len[k]) continue;                              // (min offset (count queue)): no msgs, omitted
      keys = (keys & ~(0xFFFFu << (16 * i))) | (k << (16 * i));
      a.p1 |= (uint64_t)len[k] << (32 * i);
    }
    out_type = MS_T_POLL_OK;
    a.p0 = keys;
  } else if (type == MS_T_COMMIT_OFFSETS) {                                       // merge-with max (:159-165)
    if (!kf_keys_ok(c, m.p0)) return;
    for (int i = 0; i < 2; i++) {
      const uint32_t k = (m.p0 >> (16 * i)) & 0xFFFFu, o = (uint32_t)(m.p1 >> (32 * i));
      if (k == kKafkaNoKey) continue;
      if (o == kKafkaAbsent) { latch_error(c.st, E_VALUE_RANGE, o); return; }
      if (committed[k] == kKafkaAbsent || o > committed[k]) committed[k] = o;
    }
    out_type = MS_T_COMMIT_OFFSETS_OK;
  } else if (type == MS_T_LIST_COMMITTED_OFFSETS) {                               // select-keys (:167-172)
    if (!kf_keys_ok(c, m.p0)) return;
    uint32_t keys = 0xFFFFFFFFu;
    for (int i = 0; i < 2; i++) {
      const uint32_t k = (m.p0 >> (16 * i)) & 0xFFFFu;
      if (k == kKafkaNoKey || committed[k] == kKafkaAbsent) continue;
      keys = (keys & ~(0xFFFFu << (16 * i))) | (k << (16 * i));
      a.p1 |= (uint64_t)committed[k] << (32 * i);
    }
    out_type = MS_T_LIST_COMMITTED_OFFSETS_OK;
    a.p0 = keys;
  } else {
    a.p0 = 10;                                                                    // "Unknown request type", {:code 10}
  }
  a.tf = out_type | ((has_id ? (uint32_t)MS_F_REPLY : 0u) << 16);
  rf_emit(c, a);
}

// ------------------------------------------------------------------ g-counter / pn-counter
// demo/ruby/pn_counter.rb on crdt.rb and node.rb (DESIGN.md 2.16), for both workloads.  The PN counter is two
// G-counters, maps node id -> count; a node only ever names the members of its block (node_ids of its init), so the maps
// are rows of Params.ct_val in block order: inc[0, gn) then dec at + ct_width.  Handlers run in dequeue order, a legal
// schedule of Ruby's thread per message.  RaftDev.state = 1: crashed (main! raised on a type without a handler).  The
// replication task keeps g-set's schedule (gs_init / gs_next_fire / gs_fires) and tags its snapshot rows in gs_tag.
__device__ __forceinline__ int64_t* ct_row(const Params& p, uint32_t e) { return p.ct_val + (size_t)e * 2 * p.ct_width; }

// `every 5` (crdt.rb:41-45, node.rb:129-137), at the start of the node's step: snapshot @value for run k, then
// merge to every other block member in index order
__device__ void ct_task(RaftCtx& c) {
  const Params& p = c.p;
  if (c.r->state || !p.gs_init[c.e] || c.now < p.gs_next_fire[c.e]) return;
  const uint32_t k = ++p.gs_fires[c.e];
  const size_t row = (size_t)c.e * p.gs_slots + (k & (p.gs_slots - 1u));
  const int64_t* mine = ct_row(p, c.e);
  int64_t* snap = p.ct_snap + row * 2 * p.ct_width;
  for (uint32_t i = 0; i < c.gn; i++) { snap[i] = mine[i]; snap[p.ct_width + i] = mine[p.ct_width + i]; }
  p.gs_tag[row] = k;
  for (uint32_t n = c.gbase; n < c.gbase + c.gn; n++) {
    if (n == c.e) continue;
    Rec m;                                                                        // send! (node.rb:68-78): no msg_id
    m.round = 0; m.ticket = 0; m.idx = 0;
    m.src = c.e; m.dest = n; m.msg_id = 0; m.in_reply_to = 0;
    m.tf = MS_T_MERGE; m.p0 = 0; m.p1 = k;
    rf_emit(c, m);
  }
  p.gs_next_fire[c.e] += (int64_t)p.gs_interval_ms * kTickNs;
}

__device__ void ct_handle(RaftCtx& c, const Rec& m) {
  const Params& p = c.p;
  if (c.r->state) return;                                                         // crashed: read, never acted on
  const uint32_t type = m.tf & 0xFFFFu, flags = m.tf >> 16;
  if (flags & MS_F_REPLY) return;                                                 // no callbacks (node.rb:159-164)
  if (type == MS_T_MERGE_OK) return;                                              // crdt.rb:36-38
  const bool has_id = (flags & MS_F_MSG_ID) != 0;
  Rec a;                                                                          // reply! (node.rb:88-91)
  a.round = 0; a.ticket = 0; a.idx = 0;
  a.src = c.e; a.dest = m.src; a.msg_id = 0;
  a.in_reply_to = has_id ? m.msg_id : 0u;                                         // in_reply_to: nil without a msg_id
  a.p0 = 0; a.p1 = 0;
  int64_t* mine = ct_row(p, c.e);
  const uint32_t W = p.ct_width;
  uint32_t out_type;
  if (type == MS_T_INIT) {                                                        // node.rb:22-36: (re)starts the task,
    p.gs_init[c.e] = 1;                                                           // first run in the next round
    p.gs_next_fire[c.e] = c.now;
    out_type = MS_T_INIT_OK;
  } else if (type == MS_T_ADD) {                                                  // pn_counter.rb:77-83
    const int32_t delta = (int32_t)m.p0;
    if (delta >= 0) mine[c.e - c.gbase] += delta;
    else mine[W + c.e - c.gbase] += -(int64_t)delta;
    out_type = MS_T_ADD_OK;
  } else if (type == MS_T_READ) {                                                 // crdt.rb:25-27, pn_counter.rb:71-73
    int64_t v = 0;
    for (uint32_t i = 0; i < c.gn; i++) v += mine[i] - mine[W + i];
    a.p1 = (uint64_t)v;
    out_type = MS_T_READ_OK;
  } else if (type == MS_T_MERGE) {                                                // crdt.rb:30-34: merge by max
    const uint32_t k = (uint32_t)m.p1;
    const size_t row = (size_t)m.src * p.gs_slots + (k & (p.gs_slots - 1u));
    // only a block member's task sends merges, with its run k >= 1; the row must still hold that run
    if (m.src < c.gbase || m.src >= c.gbase + c.gn || m.src == c.e || k == 0 || (uint64_t)k != m.p1 ||
        __ldcg(p.gs_tag + row) != k) {
      latch_error(c.st, E_SNAPSHOT, m.src);
      return;
    }
    const int64_t* snap = p.ct_snap + row * 2 * W;
    for (uint32_t i = 0; i < c.gn; i++) {
      mine[i] = max(mine[i], snap[i]);
      mine[W + i] = max(mine[W + i], snap[W + i]);
    }
    out_type = MS_T_MERGE_OK;
  } else {
    c.r->state = 1;                                                               // "No handler": main! raises (node.rb:167),
    p.gs_init[c.e] = 0;                                                           // the process and its task end
    return;
  }
  a.tf = out_type | ((has_id ? (uint32_t)MS_F_REPLY : 0u) << 16);
  rf_emit(c, a);
}

// ------------------------------------------------------------------ txn-rw-register
// demo/clojure/txn_rw_register_hat.clj on node.clj (DESIGN.md 2.17).  node.clj:178 parses a message with string keys
// and keywordizes only the top level and the body (:165-171), so a replicate's txn+s are string-keyed maps: apply-txn+!
// finds neither :ts nor :txn (:40) and applies an empty txn under a fresh timestamp, nothing enters the receiver's
// unreplicated map, and the acks carry nil timestamps that remove nothing (:145,157).  A node's unreplicated map is
// therefore every txn it has served, each pending at every other block member: its size is the log's length.
// RaftDev.state = 1: init received (the node-id promise is delivered).  Handlers run one at a time in dequeue order.
__device__ __forceinline__ Rec rw_msg(const RaftCtx& c, uint32_t dest, uint32_t type, uint32_t p0) {
  Rec m;                                                                          // send! (node.clj:110-115): no msg_id
  m.round = 0; m.ticket = 0; m.idx = 0;
  m.src = c.e; m.dest = dest; m.msg_id = 0; m.in_reply_to = 0;
  m.tf = type; m.p0 = p0; m.p1 = 0;
  return m;
}

// the replication thread (:104-114): (Thread/sleep 100) then replicate-step!, from process start, at the start of the
// node's step.  The node's step may come after several periods (it is only stepped when due with a non-empty log, or
// for mail): a period that passed with an empty log sent nothing, so the schedule moves on to the next period after now
__device__ void rw_task(RaftCtx& c) {
  const Params& p = c.p;
  int64_t& next = p.gs_next_fire[c.e];
  if (c.now < next) return;
  const uint32_t n = p.rw_len[c.e];
  if (n) rf_emit(c, rw_msg(c, c.gbase == c.e ? c.e + 1u : c.gbase, MS_T_REPLICATE, n));   // the lowest other member
  const int64_t period = (int64_t)p.gs_interval_ms * kTickNs;
  next += ((c.now - next) / period + 1) * period;
}

__device__ void rw_handle(RaftCtx& c, const Rec& m) {
  const Params& p = c.p;
  const uint32_t type = m.tf & 0xFFFFu, flags = m.tf >> 16;
  if (flags & MS_F_REPLY) return;                                                 // handle-reply!: no rpcs (node.clj:131-139)
  if (type != MS_T_INIT && !c.r->state) return;                                   // blocked on the node-id promise
  if (type == MS_T_REPLICATE_ACK) return;                                         // nil timestamps: nothing to remove
  const bool has_id = (flags & MS_F_MSG_ID) != 0;
  Rec a;                                                                          // reply! (node.clj:116-119)
  a.round = 0; a.ticket = 0; a.idx = 0;
  a.src = c.e; a.dest = m.src; a.msg_id = 0;
  a.in_reply_to = has_id ? m.msg_id : 0u;                                         // in_reply_to: nil without a msg_id
  a.p0 = 0; a.p1 = 0;
  uint64_t& lamport = p.rw_lamport[c.e];
  uint32_t out_type = MS_T_ERROR;
  if (type == MS_T_INIT) {                                                        // handle-init! (node.clj:141-151)
    c.r->state = 1;
    out_type = MS_T_INIT_OK;
  } else if (type == MS_T_TXN) {                                                  // txn_rw_register_hat.clj:116-125
    const uint32_t len = p.rw_len[c.e];
    for (int i = 0; i < 4; i++) {
      const uint32_t op = (uint32_t)(m.p1 >> (16 * i)) & 0xFFFFu;
      if ((op >> 15) && (op & 0x3FFFu) >= p.rw_keys) { latch_error(c.st, E_VALUE_RANGE, op & 0x3FFFu); return; }
    }
    if (len >= p.rw_cap) { latch_error(c.st, E_TXN_RW_CAPACITY, c.e); return; }
    const uint64_t ts = lamport++;                                                // apply-txn+: [lamport node-id]
    ms_txn_rw_entry en;
    en.lamport = ts; en.ops = m.p1; en.base = m.p0; en.pad = 0;
    uint32_t* val = p.rw_val + (size_t)c.e * p.rw_keys;
    uint64_t* wts = p.rw_ts + (size_t)c.e * p.rw_keys;
    for (int i = 0; i < 4; i++) {
      const uint32_t op = (uint32_t)(m.p1 >> (16 * i)) & 0xFFFFu, k = op & 0x3FFFu;
      en.reads[i] = 0;
      if (!(op >> 15)) continue;
      if (op & (1u << 14)) { val[k] = m.p0 + (uint32_t)i; wts[k] = ts; }          // a fresh ts is above every stored one
      else en.reads[i] = val[k];
    }
    p.rw_log[(size_t)c.e * p.rw_cap + len] = en;
    p.rw_len[c.e] = len + 1u;                                                     // later-replicate!
    out_type = MS_T_TXN_OK;
    a.p0 = len; a.p1 = ts;
  } else if (type == MS_T_REPLICATE) {                                            // :127-145
    lamport += m.p0;                                                              // an empty txn per txn+
    for (uint32_t n = c.gbase; n < c.gbase + c.gn; n++)
      if (n != c.e) rf_emit(c, rw_msg(c, n, MS_T_REPLICATE_ACK, m.p0));           // other-node-ids, block order
    return;
  } else {
    a.p0 = 10;                                                                    // "Unknown request type" (node.clj:155-163)
  }
  a.tf = out_type | ((has_id ? (uint32_t)MS_F_REPLY : 0u) << 16);
  rf_emit(c, a);
}

// ------------------------------------------------------------------ txn-list-append on a persistent hash tree
// demo/ruby/datomic_list_append.rb.  The database is a tree of immutable nodes stored in lww-kv under
// unique pointers; lin-kv holds the pointer to the root (key "root" = key 0 here).  A txn (:340-353, under
// @txn_lock: one at a time per node, here in arrival order): read the root pointer, load the tree lazily
// (Tree.load :83-101: cache, else read lww-kv until it answers read_ok), apply the micro-ops (path copying,
// csrc/ms_tree.h), and if the tree changed write every new node to lww-kv, wait for all write_oks, then cas the
// root from the pointer read to the new one: cas_ok -> txn_ok, anything else -> error 30.  A root that cannot
// be read is error 14 (abort, :361-368).  sync_rpc! is a blocked thread in the reference; here the node is a
// state machine and the blocked evaluation is redone after every load (same result, see ms_tree.h).
// Promise#await gives up after 5 s (promise.rb): a sync_rpc! that gets no reply raises RPCError.timeout, which the
// handler thread turns into an error 0 reply (node.rb:187-189) and which releases the lock.  save! of a Branch waits in
// a helper thread that turns a time-out into "false" (:297-309) while the handler waits 5 s for that verdict itself:
// if the first write is still unanswered when both clocks run out the helper's "false" is taken to arrive first
// (error 14, "Couldn't save new tree"), otherwise the handler's own time-out does (error 0).  A reply that arrives
// after its waiter gave up finds a dead promise: ignored.
struct TreeStore {
  const Params& p;
  uint32_t e;
  __device__ mst::Rec* rec(uint32_t ptr) const { return reinterpret_cast<mst::Rec*>(p.tt_recs) + (ptr - 1u); }
  __device__ bool cached(uint32_t ptr) const {
    const uint32_t* tab = p.tt_cache + (size_t)e * (p.tt_cache_mask + 1u);
    for (uint32_t h = (ptr * 0x9E3779B1u) & p.tt_cache_mask, n = 0; n <= p.tt_cache_mask; n++, h = (h + 1u) & p.tt_cache_mask) {
      if (tab[h] == ptr) return true;
      if (tab[h] == 0u) return false;
    }
    return false;
  }
};

__device__ void tt_cache_insert(RaftCtx& c, uint32_t ptr) {                       // @@cache[ptr] = tree, :95
  uint32_t* tab = c.p.tt_cache + (size_t)c.e * (c.p.tt_cache_mask + 1u);
  uint32_t h = (ptr * 0x9E3779B1u) & c.p.tt_cache_mask;
  for (uint32_t n = 0; n < c.p.tt_cache_mask; n++, h = (h + 1u) & c.p.tt_cache_mask) {   // one slot always stays empty
    if (tab[h] == ptr) return;
    if (tab[h] == 0u) { tab[h] = ptr; return; }
  }
  latch_error(c.st, E_RAFT_CAPACITY, c.e);
}

// Node#rpc! (node.rb:95-102): msg_id = @next_msg_id += 1, remember the handler, send
__device__ void tt_rpc(RaftCtx& c, uint32_t dest, uint32_t type, uint32_t p0, uint64_t p1, uint32_t kind, uint32_t arg) {
  if (dest == 0xFFFFFFFFu) { latch_error(c.st, E_INVALID_DEST, dest); return; }   // the workload needs lin-kv and lww-kv
  const uint32_t id = ++c.r->next_msg_id;
  uint4* slot = c.cb + 2 * (size_t)(id & c.p.rf_cb_mask);
  slot[0] = make_uint4(id, kind, arg, c.p.tt_node[c.e].gen);
  slot[1] = make_uint4(0u, 0u, 0u, 0u);
  Rec r;
  r.round = 0; r.ticket = 0; r.idx = 0;
  r.src = c.e; r.dest = dest; r.msg_id = id; r.in_reply_to = 0;
  r.tf = type | ((uint32_t)MS_F_MSG_ID << 16);
  r.p0 = p0; r.p1 = p1;
  rf_emit(c, r);
}

__device__ void tt_start(RaftCtx& c, TreeDev* t, uint32_t src, uint32_t msg_id, uint64_t ops);

__device__ void tt_finish(RaftCtx& c, TreeDev* t) {                               // @txn_lock released: the next waiter runs
  t->phase = 0;
  t->deadline = 0;
  t->gen++;
  if (t->q_head != t->q_tail) {
    const uint4 q = c.p.tt_queue[(size_t)c.e * kTreeQueue + (t->q_head % kTreeQueue)];
    t->q_head++;
    tt_start(c, t, q.x, q.y, (uint64_t)q.z | ((uint64_t)q.w << 32));
  }
}

__device__ void tt_answer(RaftCtx& c, TreeDev* t, uint32_t type, uint32_t code, uint64_t p1) {
  Rec req;
  req.round = 0; req.ticket = 0; req.idx = 0;
  req.src = t->cur_src; req.dest = c.e; req.msg_id = t->cur_msg_id; req.in_reply_to = 0; req.tf = MS_T_TXN; req.p0 = 0; req.p1 = 0;
  Rec a = rf_reply_to(c, req, type);
  a.p0 = code; a.p1 = p1;
  rf_emit(c, a);
  tt_finish(c, t);
}

__device__ void tt_start(RaftCtx& c, TreeDev* t, uint32_t src, uint32_t msg_id, uint64_t ops) {
  t->cur_src = src; t->cur_msg_id = msg_id; t->cur_ops = ops;
  t->phase = 1;
  t->deadline = c.now + kPromiseTimeoutNs;
  tt_rpc(c, c.p.sv_ep[MS_SVC_LIN_KV], MS_T_READ, 0u, 0ull, 10u, 0u);             // current_tree, :361-368
}

// tree1 -> apply_txn -> (save!, advance_root!) -> reply, as far as the node can get without another read (:340-353)
__device__ void tt_eval(RaftCtx& c, TreeDev* t) {
  TreeStore S{c.p, c.e};
  uint32_t counter = t->start_counter, root2 = 0, load_ptr = 0;
  const mst::Status st = mst::apply_txn(S, c.e, c.p.tt_per_node, t->root1, t->cur_ops, t->start_counter, counter, root2, load_ptr);
  if (st == mst::kCapacity) { latch_error(c.st, E_RAFT_CAPACITY, c.e); return; }
  if (st == mst::kNeedLoad) {                                                     // Tree.load, :83-101
    t->phase = 2; t->load_ptr = load_ptr;
    t->deadline = c.now + kPromiseTimeoutNs;
    tt_rpc(c, c.p.sv_ep[MS_SVC_LWW_KV], MS_T_READ, load_ptr, 0ull, 11u, load_ptr);
    return;
  }
  t->ptr_counter = counter;
  t->root2 = root2;
  if (root2 == t->root1) {                                                        // nothing appended: no save, no cas
    tt_answer(c, t, MS_T_TXN_OK, 0u, (uint64_t)t->root1 | ((uint64_t)t->root1 << 32));
    return;
  }
  uint32_t out[mst::kMaxWrites], n = 0;
  if (!mst::save_order(S, c.e, c.p.tt_per_node, t->start_counter, root2, out, n)) { latch_error(c.st, E_RAFT_CAPACITY, c.e); return; }
  t->phase = 3; t->writes_left = n; t->write_failed = 0;
  t->deadline = c.now + kPromiseTimeoutNs;
  t->first_write = out[0]; t->first_write_ok = 0; t->root_is_leaf = S.rec(root2)->type == 1 ? 1u : 0u;
  for (uint32_t i = 0; i < n; i++)                                                // save_this!, :128-145: value = the node's JSON
    tt_rpc(c, c.p.sv_ep[MS_SVC_LWW_KV], MS_T_WRITE, out[i], (uint64_t)out[i], 12u, out[i]);
}

__device__ void tt_handle(RaftCtx& c, const Rec& m) {
  TreeDev* t = c.p.tt_node + c.e;
  const uint32_t type = m.tf & 0xFFFFu, flags = m.tf >> 16;
  if (flags & MS_F_REPLY) {                                                       // node.rb:170-176
    uint4* slot = c.cb + 2 * (size_t)(m.in_reply_to & c.p.rf_cb_mask);
    const uint4 s0 = slot[0];
    if (s0.y == 0 || s0.x != m.in_reply_to) return;                               // "Ignoring reply ... with no callback"
    slot[0] = make_uint4(0u, 0u, 0u, 0u);
    if (s0.y >= 10 && s0.y <= 13 && (s0.w != t->gen || t->phase == 0)) return;    // its transaction is over: a dead promise
    if ((s0.y == 14 && t->init_phase != 1) || (s0.y == 15 && t->init_phase != 2)) return;
    switch (s0.y) {
      case 10:                                                                    // the root pointer
        if (type == MS_T_READ_OK) {
          t->root1 = (uint32_t)m.p1;
          t->start_counter = t->ptr_counter;
          tt_eval(c, t);
        } else {
          tt_answer(c, t, MS_T_ERROR, 14u, 0ull);                                 // RPCError.abort "Unsure how to handle", :367
        }
        return;
      case 11:                                                                    // a tree node
        if (type == MS_T_READ_OK) {
          tt_cache_insert(c, s0.z);
          tt_eval(c, t);
        } else {                                                                  // "Retrying read of tree node", :97-99
          t->deadline = c.now + kPromiseTimeoutNs;
          tt_rpc(c, c.p.sv_ep[MS_SVC_LWW_KV], MS_T_READ, s0.z, 0ull, 11u, s0.z);
        }
        return;
      case 12:                                                                    // one of save!'s writes
        if (type != MS_T_WRITE_OK) t->write_failed = 1;
        if (s0.z == t->first_write) t->first_write_ok = 1;
        if (--t->writes_left == 0) {
          if (t->write_failed) { tt_answer(c, t, MS_T_ERROR, 14u, 0ull); return; }   // "Couldn't save new tree", :347
          t->phase = 4;                                                           // advance_root!, :372-379
          t->deadline = c.now + kPromiseTimeoutNs;
          tt_rpc(c, c.p.sv_ep[MS_SVC_LIN_KV], MS_T_CAS, 0u, (uint64_t)t->root1 | ((uint64_t)t->root2 << 32), 13u, 0u);
        }
        return;
      case 13:
        if (type == MS_T_CAS_OK) tt_answer(c, t, MS_T_TXN_OK, 0u, (uint64_t)t->root1 | ((uint64_t)t->root2 << 32));
        else tt_answer(c, t, MS_T_ERROR, 30u, 0ull);                              // RPCError.txn_conflict, :378
        return;
      case 14: {                                                                  // the first node's initial state, :330-338
        Rec req;
        req.round = 0; req.ticket = 0; req.idx = 0;
        req.src = t->init_src; req.dest = c.e; req.msg_id = t->init_msg_id; req.in_reply_to = 0; req.tf = MS_T_INIT; req.p0 = 0; req.p1 = 0;
        if (type == MS_T_WRITE_OK) {
          t->init_phase = 2; t->init_deadline = c.now + kPromiseTimeoutNs;
          tt_rpc(c, c.p.sv_ep[MS_SVC_LIN_KV], MS_T_WRITE, 0u, (uint64_t)mst::kPtrEmpty, 15u, 0u);
        } else {
          t->init_phase = 0;
          Rec er = rf_reply_to(c, req, MS_T_ERROR);                               // "Couldn't write initial state"
          er.p0 = 14;
          rf_emit(c, er);
        }
        return;
      }
      case 15: {                                                                  // root written: reply! msg, type: "init_ok" (node.rb:31)
        Rec req;
        req.round = 0; req.ticket = 0; req.idx = 0;
        req.src = t->init_src; req.dest = c.e; req.msg_id = t->init_msg_id; req.in_reply_to = 0; req.tf = MS_T_INIT; req.p0 = 0; req.p1 = 0;
        t->init_phase = 0;
        rf_emit(c, rf_reply_to(c, req, MS_T_INIT_OK));
        return;
      }
    }
    return;
  }
  if (type == MS_T_INIT) {                                                        // node.rb:22-36 + :329-338
    if (c.e == 0) {                                                               // @node.node_ids.first == @node.node_id
      t->init_src = m.src; t->init_msg_id = m.msg_id;
      t->init_phase = 1; t->init_deadline = c.now + kPromiseTimeoutNs;
      tt_rpc(c, c.p.sv_ep[MS_SVC_LWW_KV], MS_T_WRITE, mst::kPtrEmpty, (uint64_t)mst::kPtrEmpty, 14u, 0u);
    } else {
      rf_emit(c, rf_reply_to(c, m, MS_T_INIT_OK));
    }
    return;
  }
  if (type == MS_T_TXN) {                                                         // :340-353
    if (t->phase == 0) { tt_start(c, t, m.src, m.msg_id, m.p1); return; }
    if (t->q_tail - t->q_head >= kTreeQueue) { latch_error(c.st, E_RAFT_CAPACITY, c.e); return; }
    c.p.tt_queue[(size_t)c.e * kTreeQueue + (t->q_tail % kTreeQueue)] = make_uint4(m.src, m.msg_id, (uint32_t)m.p1, (uint32_t)(m.p1 >> 32));
    t->q_tail++;
    return;
  }
  Rec er = rf_reply_to(c, m, MS_T_ERROR);                                         // no handler: not supported
  er.p0 = 10;
  rf_emit(c, er);
}

// Promise#await's 5 s (promise.rb:24-31), checked once per step after the step's messages: a reply that arrives in the
// round the clock runs out still counts.  k_snapshot keeps a node's ticket alive when this would act (tt_timer_due).
__device__ __forceinline__ bool tt_timer_due(const TreeDev& t, int64_t now) {
  return (t.phase != 0 && t.deadline != 0 && now >= t.deadline) || (t.init_phase != 0 && now >= t.init_deadline);
}
// The earliest instant at which tt_timer_due holds (k_wake, ms_set_idle_jump).  Keep the two in step.
__device__ __forceinline__ int64_t tt_wake_ns(const TreeDev& t) {
  int64_t w = INT64_MAX;
  if (t.phase != 0 && t.deadline != 0) w = t.deadline;
  if (t.init_phase != 0) w = min(w, t.init_deadline);
  return w;
}
__device__ void tt_actions(RaftCtx& c) {
  TreeDev* t = c.p.tt_node + c.e;
  if (t->init_phase != 0 && c.now >= t->init_deadline) {                          // the init handler's thread gives up
    t->init_phase = 0;
    Rec req;
    req.round = 0; req.ticket = 0; req.idx = 0;
    req.src = t->init_src; req.dest = c.e; req.msg_id = t->init_msg_id; req.in_reply_to = 0; req.tf = MS_T_INIT; req.p0 = 0; req.p1 = 0;
    Rec er = rf_reply_to(c, req, MS_T_ERROR);
    er.p0 = 0;                                                                    // RPCError.timeout
    rf_emit(c, er);
  }
  if (t->phase != 0 && t->deadline != 0 && c.now >= t->deadline) {
    const uint32_t code = (t->phase == 3 && !t->root_is_leaf && !t->first_write_ok) ? 14u : 0u;
    tt_answer(c, t, MS_T_ERROR, code, 0ull);                                      // releases the lock: the next waiter starts
  }
}
