/*
 * maelstrom_b200.h -- C ABI of the H100-native replacement for Maelstrom's hot
 * path: maelstrom.process (node spawn + STDIN/STDOUT pumps,
 * src/maelstrom/process.clj:68-256) and maelstrom.net (route / latency / loss /
 * partition, src/maelstrom/net.clj:79-247).  Everything above that boundary
 * (maelstrom.client, workload.*, nemesis, core, checkers) keeps calling the same
 * seven entry points; INTEGRATION.md shows the JNI / Clojure stub a maintainer
 * would add.  All paths in the comments are relative to a jepsen-io/maelstrom checkout.
 *
 * Plain C types only: no torch, no CUDA types.  The library owns all device
 * memory; callers own every out-buffer.  Any thread may call; calls on one
 * ms_sim are serialised by an internal mutex (the reference's state is one atom
 * plus thread-safe queues, net.clj:92-103).  There is NO CPU fallback: ms_create
 * fails (NULL + ms_last_error) when no CUDA device is usable.
 */
#ifndef MAELSTROM_B200_H
#define MAELSTROM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MS_ABI_VERSION 2

/* ------------------------------------------------------------------ records */

/* Message: replaces the Message record {^long id src dest body}
 * (net/message.clj:8-15).  48 bytes = three 16-byte vectors.  Node ids are dense
 * indices: servers n0..n{N-1} (core.clj:231-238) are 0..N-1, endpoints added
 * with ms_add_endpoint follow.  body = {type, msg_id, in_reply_to} (the
 * reserved keys, doc/protocol.md:36-45) + 12 payload bytes. */
typedef struct ms_msg {
  uint64_t id;          /* net id, ++next-message-id (net.clj:197); first is 0 */
  int64_t  deadline_ns; /* virtual deadline = now + latency_ms*1e6 (net.clj:202-205) */
  uint32_t src, dest;
  uint32_t msg_id;      /* body.msg_id,      valid iff flags & MS_F_MSG_ID */
  uint32_t in_reply_to; /* body.in_reply_to, valid iff flags & MS_F_REPLY  */
  uint16_t type;        /* MS_T_* */
  uint16_t flags;
  uint32_t p0;          /* payload: broadcast "message" / g-set "element" / error "code" / read_ok count */
  uint64_t p1;          /* payload: opaque 8 bytes (echo) or host blob handle */
} ms_msg;

/* Body as passed by the host data plane (client/send!, client.clj:66-79). */
typedef struct ms_body {
  uint16_t type, flags;
  uint32_t msg_id, in_reply_to, p0;
  uint64_t p1;
} ms_body;

/* Journal event: replaces Event{id time type message} (net/journal.clj:53).
 * bit 63 of event_id is the type: 0 = :send, 1 = :recv. */
typedef struct ms_event {
  uint64_t event_id;    /* ++next-id (journal.clj:228,236), dense from 0 */
  int64_t  time_ns;     /* virtual time of the round (replaces linear-time-nanos, journal.clj:229) */
  uint64_t msg_id;      /* Message.id */
  uint32_t src, dest;
} ms_event;
#define MS_EVENT_RECV (1ull << 63)

/* Body of the message of a journal event (journal level 2), 32 bytes. */
typedef struct ms_jbody {
  uint64_t id;
  uint32_t msg_id, in_reply_to;
  uint16_t type, flags;
  uint32_t p0;
  uint64_t p1;
} ms_jbody;

/* Scheduled client op: a message injected when virtual time reaches time_ns
 * (device-resident stand-in for the Jepsen generator, core.clj:67-80). */
typedef struct ms_op {
  int64_t  time_ns;
  uint32_t src, dest;
  ms_body  body;
} ms_op;

enum { MS_F_MSG_ID = 1, MS_F_REPLY = 2,
       MS_F_CREATE = 4,     /* cas: create_if_not_exists (service.clj:50-54) */
       MS_F_APPENDS = 8 };  /* txn: the micro-op list contains an append */

/* body.type codes (doc/workloads.md; SURVEY.md appendix E) */
enum {
  MS_T_INIT = 1, MS_T_INIT_OK = 2, MS_T_ERROR = 3,
  MS_T_ECHO = 10, MS_T_ECHO_OK = 11,
  MS_T_TOPOLOGY = 20, MS_T_TOPOLOGY_OK = 21, MS_T_BROADCAST = 22,
  MS_T_BROADCAST_OK = 23, MS_T_READ = 24, MS_T_READ_OK = 25,
  MS_T_ADD = 30, MS_T_ADD_OK = 31, MS_T_REPLICATE_ONE = 32, MS_T_REPLICATE_FULL = 33,
  /* services (doc/services.md, service.clj:31-141).  read = MS_T_READ with p0 = key and read_ok
   * p1 = value; write p0 = key, p1 = value; cas p0 = key, p1 = from | to << 32 (+ MS_F_CREATE);
   * ts_ok p1 = timestamp; errors: MS_T_ERROR with p0 = 20 / 22 (errors.edn).  Keys are integers
   * below ms_config.reserved[2]; values are 32-bit on the device. */
  MS_T_WRITE = 40, MS_T_WRITE_OK = 41, MS_T_CAS = 42, MS_T_CAS_OK = 43, MS_T_TS = 44, MS_T_TS_OK = 45,
  /* Raft (raft.py:270-281,405-432,460-545): request_vote p0 = term, p1 = last_log_index |
   * last_log_term << 32; *_res p0 = term, p1 = vote_granted / success; append_entries p0 = term,
   * p1 = k: the sender's k-th append_entries; {prev_log_index, prev_log_term, leader_commit,
   * entries} stay in the sender's payload heap on the device */
  MS_T_REQUEST_VOTE = 50, MS_T_REQUEST_VOTE_RES = 51, MS_T_APPEND_ENTRIES = 52, MS_T_APPEND_ENTRIES_RES = 53,
  /* txn-list-append: txn p1 = the caller's handle of the micro-op list, flag MS_F_APPENDS when it
   * contains an append; txn_ok p1 = version read | version written << 32.  Database values are
   * carried as version ids: 0 = nil (no root yet), 1 = the empty database, others minted by the
   * node whose cas installs them; the caller replays apply-txn (single_key_txn.clj:115-127) over them */
  MS_T_TXN = 60, MS_T_TXN_OK = 61
};

enum { MS_W_ECHO = 0, MS_W_BROADCAST = 1, MS_W_GSET = 2,                     /* --workload, core.clj:36-47 */
       MS_W_RAFT = 3,    /* lin-kv served by Raft nodes (demo/python/raft.py) */
       MS_W_TXN_TREE = 5,  /* txn-list-append on a persistent hash tree: immutable tree nodes in lww-kv, the root pointer in
                             lin-kv (demo/ruby/datomic_list_append.rb).  Needs the lin-kv and lww-kv services.  A txn carries
                             up to four micro-ops in p1, 16 bits each: valid << 15 | append << 14 | key (< 16384); p0 is the
                             caller's handle.  txn_ok: p1 = root pointer read | root pointer written << 32 (the caller replays
                             apply_txn over the chain of roots).  Pointer "n<e>-<p>" = 2 + e * reserved[3] + (p - 1), "empty" = 1;
                             ms_config.reserved[3] = pointers a node may mint (default 256), reserved[4] = tree nodes a node
                             may cache (default 1024), reserved[2] (service keys) defaults to cover every pointer.
                             A sync RPC without a reply times out after 5 s (promise.rb): error 0 to the client. */
       MS_W_TXN = 4 };   /* txn-list-append, whole database in one lin-kv key (demo/clojure/single_key_txn.clj);
                            needs the "lin-kv" service endpoint */
enum { MS_TOPO_GRID = 0, MS_TOPO_LINE = 1, MS_TOPO_TOTAL = 2,                /* --topology, broadcast.clj:169-178 */
       MS_TOPO_TREE2 = 3, MS_TOPO_TREE3 = 4, MS_TOPO_TREE4 = 5 };
enum { MS_DIST_CONSTANT = 0, MS_DIST_UNIFORM = 1, MS_DIST_EXPONENTIAL = 2 }; /* --latency-dist, net.clj:73-77 */
enum { MS_KIND_SERVER = 0,      /* device-resident node program (replaces process/start-node!) */
       MS_KIND_CLIENT = 1,      /* host-visible client, id "c<k>" (util.clj:7-10): zero latency */
       MS_KIND_HOST = 2,        /* host-visible non-client endpoint (a JVM service, service.clj:245-263) */
       MS_KIND_SIM_CLIENT = 3,  /* device-resident client sink (replies are counted, not mailed) */
       MS_KIND_SERVICE = 4,     /* device-resident service; the id picks it: "lin-kv", "seq-kv", "lww-kv",
                                   "lin-tso" (service/default-services, service.clj:290-296) */
       MS_KIND_GEN_CLIENT = 5 };/* device-resident closed-loop client: maelstrom.client + a Jepsen worker (ms_add_gen_clients) */
enum { MS_SVC_LIN_KV = 0, MS_SVC_SEQ_KV = 1, MS_SVC_LWW_KV = 2, MS_SVC_LIN_TSO = 3 };

/* error codes (negative returns); MS_ERR_NODE_NOT_FOUND maps to Maelstrom error
 * code 1 {:type ::node-not-found :definite? true} (net.clj:159-164) */
enum {
  MS_OK = 0,
  MS_ERR_NODE_NOT_FOUND = -1,
  MS_ERR_ARG = -2,
  MS_ERR_SIM = -3,        /* device-side fault latched; see ms_last_error */
  MS_ERR_CUDA = -4,
  MS_ERR_CAPACITY = -5
};

/* ------------------------------------------------------------------ lifecycle */

/* Replaces (net/net latency-map log-send? log-recv?) (net.clj:79-103, called once
 * from core.clj:57-59) plus the --node-count / --topology / --latency flags. */
typedef struct ms_config {
  uint32_t n_nodes;          /* --node-count */
  uint32_t workload;         /* MS_W_*: built-in transition kernel instead of --bin */
  uint32_t topology;         /* MS_TOPO_* */
  uint32_t latency_dist;     /* MS_DIST_* */
  uint32_t latency_mean_ms;  /* --latency (parse-long, core.clj:171-174) */
  uint32_t seed_lo, seed_hi; /* Philox key; the reference is unseeded */
  double   p_loss;           /* net.clj:100 starts at 0; no CLI flag upstream */
  uint32_t n_values;         /* size of the value universe (seen-set bitmap bits per node) */
  uint32_t gset_interval_ms; /* g-set replication period (demo/ruby/g_set.rb:34) */
  /* engine sizing (0 = default) */
  uint32_t max_endpoints;    /* servers + clients + services */
  uint32_t ring_cap;         /* per-endpoint inbox ring capacity, power of two */
  uint32_t max_window;       /* max messages one endpoint consumes per round (<= 8192) */
  uint32_t journal_cap_log2; /* device journal ring = 2^k events */
  uint32_t journal_level;    /* 0 off, 1 events, 2 events + bodies */
  uint32_t journal_discard;  /* 1: device journal is overwritten, never drained (kernel-only runs) */
  uint32_t calendar_slots;   /* timing-wheel slots (ticks), power of two */
  uint32_t calendar_cap;     /* messages per wheel slot */
  uint32_t mailbox_cap;      /* host-visible deliveries buffered between syncs */
  uint32_t inject_cap;       /* host sends staged per round */
  int32_t  device;           /* CUDA device ordinal */
  uint32_t threads_per_node; /* CTA size of the round kernel (0 = auto) */
  uint32_t n_shards;         /* GPUs the endpoints are sharded over (0/1 = single GPU), <= 8 */
  uint32_t shard_id;         /* this process's shard */
  uint32_t reserved[6];      /* [0] = rounds of id history to keep (0 = default); [1] = 1: replay round batches from a CUDA graph; [2] = keys per service store / Raft KV (0 = 4096); [3] = Raft log capacity per node (0 = 4096); [4] = servers per Raft cluster: node_ids of a node's init = its block of g consecutive servers (0 = all servers, one cluster); [5] = pending-RPC table slots per Raft / txn node (0 = 4096) */
  /* ABI 2.  Servers and the other endpoints (clients, hosts, services) may be sized apart: a
   * service hears from every node, a node from a few.  0 = ring_cap / max_window. */
  uint32_t server_ring_cap;  /* inbox ring capacity of the servers, power of two */
  uint32_t server_max_window;/* max messages one server consumes per round */
} ms_config;

typedef struct ms_sim ms_sim;

ms_sim*     ms_create(const ms_config* cfg);
void        ms_destroy(ms_sim* sim);
/* per-thread text of the last failure (sim may be NULL for ms_create failures) */
const char* ms_last_error(ms_sim* sim);
uint32_t    ms_abi_version(void);

/* process/start-node! (process.clj:168-215) / stop-node! (:217-256): select the
 * built-in node program for all servers / retire them. */
int ms_start_nodes(ms_sim* sim, uint32_t workload);
int ms_stop_nodes(ms_sim* sim);

/* net/add-node! / remove-node! (net.clj:139-152).  Returns the dense index. */
int ms_add_endpoint(ms_sim* sim, const char* id, int kind);
int ms_remove_endpoint(ms_sim* sim, uint32_t idx);
int ms_endpoint_index(ms_sim* sim, const char* id);   /* MS_ERR_NODE_NOT_FOUND if absent */

/* ------------------------------------------------------------------ data plane */

/* net/send! (net.clj:189-221) for host-visible endpoints.  The message is sent at
 * the start of the next round, in call order.  Returns the net id it will get,
 * or MS_ERR_NODE_NOT_FOUND (net.clj:172-175). */
int64_t ms_send(ms_sim* sim, uint32_t src, uint32_t dest, const ms_body* body);

/* net/recv! (net.clj:223-247): 1 = message delivered into *out, 0 = virtual
 * timeout elapsed, <0 error.  Advances the simulation while waiting. */
int ms_recv(ms_sim* sim, uint32_t endpoint, int64_t timeout_virtual_ns, ms_msg* out);

/* The same two calls with the protocol's JSON envelope (doc/protocol.md:36-45), for callers that hold what a
 * node process prints and reads.  ms_send_json = process/parse-msg + net/check-message (process.clj:26-66,
 * net.clj:27-37: {"src","dest","body"} + optional integer "id", nothing else; a malformed line is MS_ERR_ARG
 * with the reference's message) + net/send!.  ms_recv_json = net/recv! + the line process/stdin-thread would
 * write (process.clj:162): {"id","src","dest","body"} with the body's keys sorted; returns 1 / 0 / <0 like
 * ms_recv.  Payloads the device does not interpret (an echo string, a txn's micro-ops, extra keys) are kept
 * on the host and re-attached on delivery. */
int64_t ms_send_json(ms_sim* sim, const char* line);
int     ms_recv_json(ms_sim* sim, uint32_t endpoint, int64_t timeout_virtual_ns, char* out, size_t cap);

/* Closed-loop clients on the device (SURVEY.md 8f NEXT-2): what a Jepsen worker does with
 * maelstrom.client (client.clj:41-172) and the workload's generator (workload/broadcast.clj:187-241,
 * core.clj:67-80), as a per-client state machine that runs inside the round kernel:
 *   one outstanding request per client (client.clj:69-76), msg_id from 1 (:52,61-64), a reply whose
 *   in_reply_to is not the awaited id is discarded (:106-107), timeout_ns of virtual time without the
 *   reply ends the op as :info -- :fail for reads, which are idempotent (:160-164) -- error replies are
 *   :fail when the code is definite (all but 0 and 13, resources/errors.edn) else :info (:165-172);
 *   ops are a mix of `broadcast` of a fresh value and `read` (g-set: `add` / `read`), staggered by a
 *   uniform delay on [0, 2 interval) (gen/stagger of 1/rate); at time_limit_ns the mix stops and after
 *   quiet_ns more every client does one final read (broadcast.clj:237-240, core.clj:75-80).
 * Client k is bound to server k mod n_nodes, draws from its own Philox stream, and its j-th broadcast
 * carries the value k + n_clients * j (unique, as the generator's 0, 1, 2, ... are).
 * Every invocation and completion is a 32-byte history record; ms_history_drain hands them over in
 * (time, round, client) order -- the Jepsen history a checker (set-full) works on.  A read's value is
 * the node's set at that moment: the record carries its size, the members of a FINAL read are what
 * ms_node_set returns once the run is over (nothing changes after the final reads). */
typedef struct ms_gen_config {
  uint32_t n_clients;
  uint32_t read_permille;    /* share of reads in the mix, out of 1000 (gen/mix: 500) */
  int64_t  interval_ns;      /* mean delay between two ops of one client (1 / rate x clients) */
  int64_t  timeout_ns;       /* 0 = 5 000 ms (client.clj:18-20) */
  int64_t  time_limit_ns;    /* --time-limit */
  int64_t  quiet_ns;         /* 0 = 10 000 ms before the final reads (core.clj:75-78) */
} ms_gen_config;
typedef struct ms_hist {
  int64_t  time_ns;
  uint64_t order;            /* round << 24 | client ordinal: sorts records of the same instant */
  uint32_t client;           /* endpoint index */
  uint32_t op;               /* the client's op counter: an invocation and its completion share it */
  uint8_t  type;             /* MS_H_INVOKE / OK / FAIL / INFO */
  uint8_t  f;                /* MS_HF_BROADCAST (g-set: add) / MS_HF_READ */
  uint16_t error;            /* completion by an error reply: its code; MS_H_TIMEOUT for :net-timeout */
  uint32_t value;            /* broadcast / add: the value; read ok: the size of the set returned */
} ms_hist;
enum { MS_H_INVOKE = 0, MS_H_OK = 1, MS_H_FAIL = 2, MS_H_INFO = 3, MS_H_TIMEOUT = 0xFFFF };
enum { MS_HF_BROADCAST = 0, MS_HF_READ = 1 };
/* adds cfg->n_clients endpoints "c<first_name> ..." and returns the index of the first; once per simulation */
int ms_add_gen_clients(ms_sim* sim, const ms_gen_config* cfg, uint32_t first_name);
int ms_history_drain(ms_sim* sim, ms_hist* out, size_t cap, size_t* n_out);

/* Upload a time-sorted schedule of client ops (appends). */
int ms_schedule_ops(ms_sim* sim, const ms_op* ops, size_t n);

/* ------------------------------------------------------------------ time */
int      ms_step(ms_sim* sim, uint64_t n_rounds);       /* exactly n rounds */
int      ms_run(ms_sim* sim, int64_t until_virtual_ns); /* rounds while now < until */
int64_t  ms_now(ms_sim* sim);
uint64_t ms_round(ms_sim* sim);

/* ------------------------------------------------------------------ faults: jepsen-net (net.clj:105-122) */
int ms_net_drop(ms_sim* sim, uint32_t src, uint32_t dest);   /* partitions[dest] += src */
int ms_net_heal(ms_sim* sim);
int ms_net_slow(ms_sim* sim);                                /* latency x10, stackable */
int ms_net_fast(ms_sim* sim);                                /* unwrap one level; no-op when unscaled */
int ms_net_flaky(ms_sim* sim);                               /* p-loss = 0.5 */
/* additions with no upstream equivalent (SURVEY.md section 8b) */
int ms_net_set_loss(ms_sim* sim, double p);
/* Bulk partition: endpoints i, j < n with different component ids cannot hear each other (both
 * directions, checked at dequeue like drop!).  Endpoints >= n, or listed as 0xFFFFFFFF, are never
 * cut.  Cleared by ms_net_heal. */
int ms_net_partition(ms_sim* sim, const uint32_t* component_id, size_t n);

/* ------------------------------------------------------------------ journal: jepsen-os + net.journal */
/* j/journal + j/close! (net.clj:128-137): stream drained events to a file.  A path ending in
 * ".fressian" gets the reference's own format -- Fressian `Event{id time type message}` objects as
 * net/journal.clj:55-92 writes them, one stripe (net-journal/0.fressian), needs journal_level 2 --
 * anything else the raw ms_event / ms_jbody records behind a 16-byte header. */
int ms_journal_open(ms_sim* sim, const char* path);
int ms_journal_close(ms_sim* sim);
/* Copy the next events (event_id order) into caller buffers; bodies may be NULL. */
int ms_journal_drain(ms_sim* sim, ms_event* events, ms_jbody* bodies, size_t cap, size_t* n_out);
uint64_t ms_journal_written(ms_sim* sim);

/* Streaming the journal to a throughput-bound consumer (the writer side of net/journal.clj:205-239).
 * ms_run_streamed advances the simulation like ms_run and hands the journal over in batches while the
 * next rounds are already running: the device packs events, in event-id order, into staging buffers
 * that the copy engine moves into pinned host memory (two buffers in turn), and `sink` is called once
 * per batch from the calling thread (rounds of batch i, copy of batch i-1 and the sink on batch i-2
 * overlap).  Event k of a batch has event id first_event + k; its round
 * (hence its virtual time) is the last row of `rounds` whose ev_base is <= that id.
 *   MS_JFMT_EVENT  32-B ms_event, as ms_journal_drain returns them
 *   MS_JFMT_12     96 bits: id (47) | recv (1) in words 0-1, src (24) and dest (24) in words 1-2:
 *                  w0 = id[31:0]; w1 = id[46:32] | recv << 15 | src[15:0] << 16; w2 = src[23:16] | dest << 8
 *   MS_JFMT_8      64 bits: recv << 63 | src << 47 | dest << 31 | (id - id_ref of the round); needs
 *                  endpoint indices < 65536 and every message received within 2^30 ids of the newest
 *                  one: otherwise the batch header has overflow = 1 and the call fails with MS_ERR_CAPACITY
 *   MS_JFMT_4      32 bits: a :send is 0 << 31 | src << 16 | dest -- sends appear in the journal in id order (the two
 *                  counters of net.clj:197 and journal.clj:228 run in step), so the j-th send of a round has id
 *                  id_ref + j (id_ref of an MS_JFMT_4 row = the round's first id); a :recv is 1 << 31 | (id_ref - 1 - id)
 *                  -- its src and dest are those of the :send with that id, earlier in the stream.  Needs
 *                  src < 32768, dest < 65536 and receives within 2^31 ids (else overflow, as above); one GPU
 *                  (sharded runs hand over MS_JFMT_16).  Expanding it takes the stream's history: ms_jdecoder.
 * ms_journal_decode expands a batch into ms_event records (lazily, on the host); a sharded batch comes
 * out in the order it was packed (sort by event_id, or scatter by event_id - first_event, to merge shards). */
enum { MS_JFMT_EVENT = 32, MS_JFMT_12 = 12, MS_JFMT_8 = 8, MS_JFMT_4 = 4,
       MS_JFMT_16 = 16 };  /* what a sharded run hands over for MS_JFMT_8 / MS_JFMT_12: {event id | recv << 63, the MS_JFMT_8 word} */
typedef struct ms_jround {   /* one row per round that has events in the batch */
  uint64_t round;
  int64_t  time_ns;          /* Event.time of every event of the round */
  uint64_t ev_base;          /* event id of the round's first event */
  uint64_t id_ref;           /* MS_JFMT_8: message id = id_ref + the record's low 31 bits */
} ms_jround;
typedef struct ms_jbatch {
  uint64_t first_event, n_events;
  uint64_t n_rounds;
  int64_t  now;              /* simulation state when the batch was cut */
  uint64_t round, next_event;
  uint32_t format, overflow, more, error;
  uint64_t range_events;     /* events [first_event, first_event + range_events) are covered by this batch; == n_events on
                                one GPU.  Sharded runs: n_events counts this shard's events only, in no particular order,
                                each with its event id (MS_JFMT_16, or MS_JFMT_EVENT); the shards' batches partition the range */
} ms_jbatch;
typedef int (*ms_journal_sink)(void* ctx, const ms_jbatch* batch, const ms_jround* rounds, const void* events);
/* buf_events = capacity of each of the two host buffers in events (0 = 1 << 24).  A non-zero return
 * of `sink` stops the run (MS_ERR_ARG).  Returns 0 when `until_virtual_ns` is reached. */
int ms_run_streamed(ms_sim* sim, int64_t until_virtual_ns, int format, size_t buf_events,
                    ms_journal_sink sink, void* ctx);
int ms_journal_decode(const ms_jbatch* batch, const ms_jround* rounds, const void* events, ms_event* out);
/* Stateful expansion for MS_JFMT_4 (any other format goes through as with ms_journal_decode): the decoder
 * remembers src / dest of the last 2^log2_window sends (16 B each).  Feed it the batches in stream order;
 * events obtained another way in between (ms_journal_drain) are told to it with ms_jdecoder_note.  A :recv
 * whose :send it has not seen, or a batch that starts inside a round it has not followed, is MS_ERR_ARG
 * (ms_jdecoder_error has the text). */
typedef struct ms_jdecoder ms_jdecoder;
ms_jdecoder* ms_jdecoder_create(uint32_t log2_window);
void ms_jdecoder_destroy(ms_jdecoder* dec);
int ms_jdecoder_decode(ms_jdecoder* dec, const ms_jbatch* batch, const ms_jround* rounds, const void* events, ms_event* out);
int ms_jdecoder_note(ms_jdecoder* dec, const ms_event* events, size_t n);
const char* ms_jdecoder_error(const ms_jdecoder* dec);

/* net.checker/basic-stats (net/checker.clj:28-41) folded on the device:
 * out[9] = {all, clients, servers} x {send-count, recv-count, msg-count}. */
int ms_stats(ms_sim* sim, uint64_t out[9]);

/* ------------------------------------------------------------------ node state read-back */
size_t   ms_node_set(ms_sim* sim, uint32_t node, uint32_t* values, size_t cap);
uint64_t ms_client_replies(ms_sim* sim);
/* Sends whose src or dest was not a registered endpoint when they were made (a reply to a closed
 * client, gossip to a stopped node).  The reference's assert (net.clj:166-176) throws only inside
 * the sending node's stdout thread (process.clj:148-150): the id is consumed, the network keeps
 * running.  Here the :send is journaled, the message dropped and counted; a warning, not an error. */
uint64_t ms_undeliverable(ms_sim* sim);
/* MS_W_RAFT: out = {state (0 nascent, 1 follower, 2 candidate, 3 leader), current_term,
 * voted_for + 1, commit_index, last_applied, leader + 1, log size, keys in the KV store}
 * (the fields of RaftNode, demo/python/raft.py:196-221) */
int      ms_raft_state(ms_sim* sim, uint32_t node, uint64_t out[8]);

/* device-side counters for roofline accounting: out = {rounds, sends, recvs,
 * kernel launches, lost, partition_drops, max_window, windows that needed the full sort} */
int ms_counters(ms_sim* sim, uint64_t out[8]);

/* inbox ring occupancy of the servers (n_nodes = S), as the last round left it: out = six arrays of S
 * entries {tail, limit, head} of the 48-B ring, then {tail, limit, head} of the 16-B compact gossip ring
 * (broadcast only, zero otherwise).  tail counts claimed records, [head, limit) is the window the
 * last snapshot froze, tail - limit records are still pending.  The counters are 32-bit and wrap;
 * servers another shard owns read 0.  n = capacity of out in entries (>= 6 S); returns S. */
int ms_ring_counters(ms_sim* sim, uint64_t* out, uint32_t n);

/* Start a fresh simulation as if `round` rounds, `msg_id` messages and `event_id` journal events had
 * already happened, with the inbox counters (tail / limit / head, both ring parts) of endpoint e at
 * ring_pos + e * ring_stride (mod 2^32).  For testing the engine across the 32-bit boundaries of its
 * counters.  Virtual time stays 0, journal positions stay 0-based (event ids become event_id + position).
 * Valid only before the first send, schedule or round; endpoints may exist already.  Rejects
 * round >= 2^39 (the (round << 24) | ticket order key) and msg_id or event_id >= 2^62 with MS_ERR_ARG.
 * Sharded runs: call it on every shard with the same arguments; each sets its own endpoints. */
int ms_set_origin(ms_sim* sim, uint64_t round, uint64_t msg_id, uint64_t event_id, uint32_t ring_pos,
                  uint32_t ring_stride);

/* ------------------------------------------------------------------ multi-GPU (one process per GPU)
 * Endpoints are sharded by index range; every shard runs the same rounds in lock step.
 * A message for an endpoint of another shard is written by the sending kernel straight
 * into the owner's inbox ring over NVLink peer memory (CUDA IPC), so the only per-round
 * collectives are two barriers, which the host adapter supplies:
 *   ms_shard_handles  -> opaque blob (MS_SHARD_BLOB_BYTES) describing this shard's memory
 *   ms_shard_connect  <- the blob of every peer (exchanged by the caller, e.g. all_gather)
 *   ms_set_barrier    <- optional callback(ctx, cuda_stream) that enqueues a cross-shard barrier
 *                        (e.g. a 1-element NCCL all-reduce) on the given CUDA stream; without it
 *                        the engine uses its own barrier kernel over NVLink peer flags
 * ms_stream returns the CUDA stream the engine launches on.  In sharded runs ms_journal_drain
 * fills only the events of this shard's endpoints; the other slots are 0xFF bytes. */
#define MS_SHARD_BLOB_BYTES 512
typedef void (*ms_barrier_fn)(void* ctx, void* cuda_stream);
int   ms_shard_handles(ms_sim* sim, void* blob_out);
int   ms_shard_connect(ms_sim* sim, uint32_t peer, const void* blob);
int   ms_set_barrier(ms_sim* sim, ms_barrier_fn fn, void* ctx);
void* ms_stream(ms_sim* sim);
/* pure helper: shard that owns endpoint `e` (servers: contiguous index ranges; others round-robin) */
uint32_t ms_shard_owner(uint32_t e, uint32_t n_servers, uint32_t n_shards);

/* Device-side timing on the engine's own CUDA stream (what bench.py reports):
 * ms_timer_begin records an event; ms_timer_end records another, synchronises and
 * returns the GPU milliseconds between them.  ms_profile(1) additionally brackets
 * every round-kernel launch with events; ms_profile_read returns and resets the
 * accumulated round-kernel milliseconds and launch count. */
int ms_timer_begin(ms_sim* sim);
int ms_timer_end(ms_sim* sim, double* elapsed_ms);
int ms_profile(ms_sim* sim, int enable);
int ms_profile_read(ms_sim* sim, double* round_kernel_ms, uint64_t* launches);
/* Diagnostic: per-phase SM-cycle sums of the round kernel, [4 size classes][16]:
 * slots 0-8 = ticket fetch, load, ordering, dedupe, count+scan, claims, emit,
 * epilogue, commit; slot 15 = tickets processed.  enable=1 starts accounting;
 * every call returns the sums since the previous call and clears them. */
int ms_debug_phase_cycles(ms_sim* sim, int enable, uint64_t out[64]);

/* pure helper: neighbors of `node` under workload/broadcast.clj:40-178 */
size_t ms_topology(uint32_t topology, uint32_t n, uint32_t node, uint32_t* out, size_t cap);

#ifdef __cplusplus
}
#endif
#endif
