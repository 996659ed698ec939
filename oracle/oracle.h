/*
 * oracle/oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement of the maelstrom.net + maelstrom.process hot path
 * (the reference's src/maelstrom/net.clj, net/message.clj, util.clj,
 * net/journal.clj:53,225-239, workload/broadcast.clj:40-178) together with the
 * canonical node programs (demo/ruby/echo.rb:28-40, the tutorial broadcast
 * node doc/03-broadcast/01-broadcast.md:527-544 + 02-performance.md:61-67,
 * demo/ruby/g_set.rb:13-39, demo/python/raft.py, demo/clojure/single_key_txn.clj)
 * and services (src/maelstrom/service.clj), under the deterministic refinement
 * recorded in DESIGN.md section 2 ("the spec").
 *
 * PARITY STATUS: the reference hot path is nondeterministic and has no tests
 * (SURVEY.md fact 2/3), and no JVM exists here, so the *delivery order* part
 * of this oracle is "parity unpinned": it is pinned only by the source text of
 * net.clj and by the doc/test known-answer vectors listed in
 * tests/test_oracle_golden.py (topologies, flood counts, echo counts, error
 * codes, Philox KAT vectors).  Pinned harder: the services, to the properties of
 * the reference's own test/maelstrom/service_test.clj (tests/test_oracle_services.py);
 * the Raft node, to message traces of the reference's demo/python/raft.py executed
 * here unmodified (tests/test_raft_reference.py, tests/golden/raft_reference_harness.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this library.  The product
 * (maelstrom_b200/) never links, imports or calls it.
 *
 * The struct layouts below are restated from the spec on purpose (they are
 * NOT included from include/maelstrom_b200.h) so that the oracle stays an
 * independent statement of the wire/record formats.
 */
#ifndef MAELSTROM_ORACLE_H
#define MAELSTROM_ORACLE_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 48-byte message record (SURVEY.md section 8a row H1; net/message.clj:8). */
typedef struct or_msg {
  uint64_t id;          /* net-assigned message id (net.clj:197), first id 0 */
  int64_t  deadline_ns; /* virtual delivery deadline (net.clj:202-205)       */
  uint32_t src, dest;   /* dense endpoint indices                            */
  uint32_t msg_id;      /* body.msg_id      (valid iff flags&1)              */
  uint32_t in_reply_to; /* body.in_reply_to (valid iff flags&2)              */
  uint16_t type;        /* body.type code, see OR_T_*                        */
  uint16_t flags;
  uint32_t p0;          /* payload word (value / element / error code / ...) */
  uint64_t p1;          /* payload (opaque 8 bytes / blob handle)            */
} or_msg;

/* 32-byte journal event (net/journal.clj:53). bit 63 of event_id = recv. */
typedef struct or_event {
  uint64_t event_id;
  int64_t  time_ns;
  uint64_t msg_id;
  uint32_t src, dest;
} or_event;

typedef struct or_body {
  uint16_t type, flags;
  uint32_t msg_id, in_reply_to, p0;
  uint64_t p1;
} or_body;

typedef struct or_op {      /* scheduled client op: message injected at time_ns */
  int64_t  time_ns;
  uint32_t src, dest;
  or_body  body;
} or_op;

typedef struct or_config {
  uint32_t n_nodes;         /* servers n0..n{N-1}  (core.clj:231-238)        */
  uint32_t workload;        /* OR_W_*                                        */
  uint32_t topology;        /* OR_TOPO_*                                     */
  uint32_t latency_dist;    /* OR_DIST_*  (net.clj:73-77)                    */
  uint32_t latency_mean_ms; /* --latency is parse-long, core.clj:171-174     */
  uint32_t seed_lo, seed_hi;
  double   p_loss;          /* initial loss probability (net.clj:100 => 0)   */
  uint32_t n_values;        /* capacity of the per-node value universe       */
  uint32_t gset_interval_ms;/* g-set replication period (g_set.rb:30: 5 s)   */
  uint32_t raft_group;      /* servers per Raft cluster = node_ids of a node's init (raft.py:447-459): blocks of
                               raft_group consecutive servers; 0 = one cluster of all servers                  */
  uint32_t rpc_table;       /* pending-RPC closures kept per Raft / txn node (0 = 4096; the reference's dict is unbounded) */
  uint32_t tree_ptrs;       /* OR_W_TXN_TREE: pointers a node may mint (0 = 256); pointer "n<e>-<p>" = 2 + e * tree_ptrs + (p - 1) */
} or_config;

enum { OR_W_ECHO = 0, OR_W_BROADCAST = 1, OR_W_GSET = 2,
       OR_W_RAFT = 3,     /* lin-kv workload served by Raft nodes (demo/python/raft.py) */
       OR_W_TXN = 4,      /* txn-list-append, whole database in one lin-kv key (demo/clojure/single_key_txn.clj) */
       OR_W_TXN_TREE = 5 };  /* txn-list-append on a persistent hash tree in lww-kv + a root pointer in lin-kv
                                (demo/ruby/datomic_list_append.rb); tree arithmetic: maelstrom_b200/csrc/ms_tree.h */
enum { OR_TOPO_GRID = 0, OR_TOPO_LINE = 1, OR_TOPO_TOTAL = 2,
       OR_TOPO_TREE2 = 3, OR_TOPO_TREE3 = 4, OR_TOPO_TREE4 = 5 };
enum { OR_DIST_CONSTANT = 0, OR_DIST_UNIFORM = 1, OR_DIST_EXPONENTIAL = 2 };
enum { OR_KIND_SERVER = 0, OR_KIND_CLIENT = 1, OR_KIND_HOST = 2, OR_KIND_SIM_CLIENT = 3,
       OR_KIND_SERVICE = 4,    /* lin-kv / seq-kv / lww-kv / lin-tso by name (service.clj:290-296) */
       OR_KIND_GEN_CLIENT = 5 }; /* closed-loop client: maelstrom.client + a Jepsen worker (or_add_gen_clients) */
enum { OR_SVC_LIN_KV = 0, OR_SVC_SEQ_KV = 1, OR_SVC_LWW_KV = 2, OR_SVC_LIN_TSO = 3 };
enum {
  OR_T_INIT = 1, OR_T_INIT_OK = 2, OR_T_ERROR = 3,
  OR_T_ECHO = 10, OR_T_ECHO_OK = 11,
  OR_T_TOPOLOGY = 20, OR_T_TOPOLOGY_OK = 21, OR_T_BROADCAST = 22,
  OR_T_BROADCAST_OK = 23, OR_T_READ = 24, OR_T_READ_OK = 25,
  OR_T_ADD = 30, OR_T_ADD_OK = 31, OR_T_REPLICATE_ONE = 32,
  OR_T_REPLICATE_FULL = 33,
  /* services (service.clj:31-141): read = OR_T_READ with p0 = key, read_ok p1 = value;
   * write p0 = key, p1 = value; cas p0 = key, p1 = from | to << 32; ts_ok p1 = ts */
  OR_T_WRITE = 40, OR_T_WRITE_OK = 41, OR_T_CAS = 42, OR_T_CAS_OK = 43, OR_T_TS = 44, OR_T_TS_OK = 45,
  /* Raft (raft.py:270-281,405-432,460-545): request_vote p0 = term, p1 = last_log_index |
   * last_log_term << 32; *_res p0 = term, p1 = vote_granted / success; append_entries p0 = term,
   * p1 = k, the sender's k-th append_entries, naming {prev_log_index, prev_log_term,
   * leader_commit, entries} (or_raft_append) */
  OR_T_REQUEST_VOTE = 50, OR_T_REQUEST_VOTE_RES = 51, OR_T_APPEND_ENTRIES = 52, OR_T_APPEND_ENTRIES_RES = 53,
  /* txn-list-append: txn p1 = handle of the micro-op list (host side), flag OR_F_APPENDS when it
   * appends; txn_ok p1 = version read | version written << 32.  Database values travel as
   * version ids: 0 = nil (no root yet), 1 = the empty database, others minted by the writer. */
  OR_T_TXN = 60, OR_T_TXN_OK = 61
};
enum { OR_F_MSG_ID = 1, OR_F_REPLY = 2, OR_F_CREATE = 4 /* cas create_if_not_exists */,
       OR_F_APPENDS = 8 /* txn contains an append */ };

typedef struct or_sim or_sim;

or_sim*  or_create(const or_config* cfg);
/* Tree.hash of demo/ruby/datomic_list_append.rb:59-61 as ms_tree.h computes it (known-answer tests) */
uint32_t or_tree_key_hash(uint32_t key);
void     or_destroy(or_sim*);
const char* or_last_error(or_sim*);

int      or_add_endpoint(or_sim*, const char* name, int kind);
int      or_remove_endpoint(or_sim*, uint32_t idx);
int64_t  or_send(or_sim*, uint32_t src, uint32_t dest, const or_body* b);
int      or_schedule(or_sim*, const or_op* ops, size_t n);
int      or_step(or_sim*, uint64_t n_rounds);
int      or_run(or_sim*, int64_t until_ns);
int      or_recv(or_sim*, uint32_t endpoint, int64_t timeout_ns, or_msg* out);
int64_t  or_now(or_sim*);
uint64_t or_round(or_sim*);
/* Start a fresh simulation at round `round`, message id `msg_id` and journal event id `event_id` (the engine's
 * ms_set_origin without its ring counters, which the oracle does not have).  Journal positions
 * (or_journal_copy's `first`) stay 0-based. */
int      or_set_origin(or_sim*, uint64_t round, uint64_t msg_id, uint64_t event_id);

int      or_net_drop(or_sim*, uint32_t src, uint32_t dest);
int      or_net_heal(or_sim*);
int      or_net_slow(or_sim*);
int      or_net_fast(or_sim*);
int      or_net_flaky(or_sim*);
int      or_net_set_loss(or_sim*, double p);
int      or_net_partition(or_sim*, const uint32_t* component, size_t n);

size_t   or_journal_size(or_sim*);
size_t   or_journal_copy(or_sim*, size_t first, or_event* ev, or_body* bodies, size_t cap);
/* 9 counters: {all,clients,servers} x {send,recv,msg}  (net/checker.clj:28-41) */
void     or_stats(or_sim*, uint64_t out[9]);
size_t   or_node_set(or_sim*, uint32_t node, uint32_t* vals, size_t cap);
size_t   or_read_snapshot(or_sim*, uint64_t msg_id, uint32_t* vals, size_t cap);
/* Closed-loop clients (client.clj:41-172 + the generator of workload/broadcast.clj:187-241, core.clj:67-80):
 * one outstanding request, msg ids from 1, stale replies discarded, timeout, error -> :fail / :info,
 * a mix of broadcast (g-set: add) and read staggered uniformly on [0, 2 interval), final reads after a
 * quiet period.  Same record layouts as the engine's ms_gen_config / ms_hist (restated). */
typedef struct or_gen_config {
  uint32_t n_clients, read_permille;
  int64_t  interval_ns, timeout_ns, time_limit_ns, quiet_ns;
} or_gen_config;
typedef struct or_hist {
  int64_t  time_ns;
  uint64_t order;
  uint32_t client, op;
  uint8_t  type, f;          /* type: 0 invoke, 1 ok, 2 fail, 3 info; f: 0 broadcast / add, 1 read */
  uint16_t error;            /* error code of the reply, 0xFFFF = timeout */
  uint32_t value;
} or_hist;
int      or_add_gen_clients(or_sim*, const or_gen_config*, uint32_t first_name);
size_t   or_history_copy(or_sim*, size_t first, or_hist* out, size_t cap);
uint64_t or_client_replies(or_sim*);
uint64_t or_undeliverable(or_sim*);   /* sends dropped because src / dest was not a registered endpoint */

/* Raft node inspection: out[0..7] = state (0 nascent, 1 follower, 2 candidate, 3 leader), term,
 * voted_for + 1, commit_index, last_applied, leader + 1, log size, kv entries */
int      or_raft_state(or_sim*, uint32_t node, uint64_t out[8]);
/* the payload of append_entries k of `sender`: out[0..3] = prev_log_index, prev_log_term,
 * leader_commit, n_entries; returns 0 when unknown */
int      or_raft_append(or_sim*, uint32_t sender, uint64_t k, uint32_t out[4]);

/* A service on its own, driven like the reference's unit test drives handle!
 * (test/maelstrom/service_test.clj:6-53): `rnd` is the 32-bit draw standing in for rand-int. */
typedef struct or_service or_service;
or_service* or_service_new(int svc_type, uint32_t buffer_size);
void     or_service_free(or_service*);
/* returns 1 and fills the reply (type, p0, p1) or 0 when the service throws (unknown request) */
int      or_service_handle(or_service*, uint32_t client, const or_body* req, uint32_t rnd, or_body* reply);

/* pure helpers, exported so the tests can pin them to golden vectors */
size_t   or_topology(uint32_t topo, uint32_t n, uint32_t node, uint32_t* out, size_t cap);
void     or_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]);
uint64_t or_latency_draw(uint32_t dist, uint32_t mean_ms, uint32_t scale,
                         const uint32_t x[4]);
uint64_t or_loss_threshold(double p);

#ifdef __cplusplus
}
#endif
#endif
