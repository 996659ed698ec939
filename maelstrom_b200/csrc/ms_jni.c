/*
 * ms_jni.c -- JNI translation unit over the C ABI (include/maelstrom_b200.h): one native per ABI
 * entry point, for the Clojure namespace integration/clojure/maelstrom/net.clj (the drop-in for
 * src/maelstrom/net.clj:79-247) and integration/java/maelstrom/b200/Native.java.
 *
 * This image has no JDK: under a compiler that cannot find <jni.h> the unit is empty, so it is part
 * of every build without breaking it.  With a JDK:
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude \
 *       maelstrom_b200/csrc/ms_jni.c -Lmaelstrom_b200 -lmaelstrom_b200 -o libms_jni.so
 * tests/test_boundary_files.py type-checks it against a minimal stand-in for jni.h
 * (tests/native/jni_stub, test infrastructure) and checks that every symbol of the header has its
 * native here and its declaration in Native.java.
 *
 * Conventions: a simulation handle is a jlong; records cross as direct ByteBuffers in the C layout
 * (little endian: ms_msg 48 B, ms_body 24 B, ms_op 40 B, ms_event 32 B, ms_jbody 32 B); negative
 * returns are the MS_ERR_* codes, the text is lastError().
 */
#if defined(__has_include)
#if __has_include(<jni.h>)
#define MS_HAVE_JNI 1
#endif
#endif

#ifdef MS_HAVE_JNI
#include <jni.h>
#include <stdint.h>
#include <string.h>
#include "maelstrom_b200.h"

#define H(h) ((ms_sim*)(intptr_t)(h))
#define FN(name) JNIEXPORT JNICALL Java_maelstrom_b200_Native_##name
#define BUF(b) ((b) ? (*env)->GetDirectBufferAddress(env, (b)) : NULL)

jint FN(abiVersion)(JNIEnv* env, jclass c) { (void)env; (void)c; return (jint)ms_abi_version(); }

/* cfg = direct ByteBuffer holding an ms_config (the Clojure side fills it field by field) */
jlong FN(create)(JNIEnv* env, jclass c, jobject cfg) {
  (void)c;
  return (jlong)(intptr_t)ms_create((const ms_config*)BUF(cfg));
}
void FN(destroy)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; ms_destroy(H(h)); }
jstring FN(lastError)(JNIEnv* env, jclass c, jlong h) { (void)c; return (*env)->NewStringUTF(env, ms_last_error(H(h))); }

jint FN(startNodes)(JNIEnv* env, jclass c, jlong h, jint workload) { (void)env; (void)c; return ms_start_nodes(H(h), (uint32_t)workload); }
jint FN(stopNodes)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return ms_stop_nodes(H(h)); }

jint FN(addEndpoint)(JNIEnv* env, jclass c, jlong h, jstring id, jint kind) {
  (void)c;
  const char* s = (*env)->GetStringUTFChars(env, id, 0);
  const int rc = ms_add_endpoint(H(h), s, kind);
  (*env)->ReleaseStringUTFChars(env, id, s);
  return rc;
}
jint FN(removeEndpoint)(JNIEnv* env, jclass c, jlong h, jint idx) { (void)env; (void)c; return ms_remove_endpoint(H(h), (uint32_t)idx); }
jint FN(endpointIndex)(JNIEnv* env, jclass c, jlong h, jstring id) {
  (void)c;
  const char* s = (*env)->GetStringUTFChars(env, id, 0);
  const int rc = ms_endpoint_index(H(h), s);
  (*env)->ReleaseStringUTFChars(env, id, s);
  return rc;
}

/* net/send! (net.clj:189-221) */
jlong FN(send)(JNIEnv* env, jclass c, jlong h, jint src, jint dest, jint type, jint flags, jint msgId,
               jint inReplyTo, jint p0, jlong p1) {
  (void)env; (void)c;
  ms_body b;
  b.type = (uint16_t)type; b.flags = (uint16_t)flags; b.msg_id = (uint32_t)msgId;
  b.in_reply_to = (uint32_t)inReplyTo; b.p0 = (uint32_t)p0; b.p1 = (uint64_t)p1;
  return ms_send(H(h), (uint32_t)src, (uint32_t)dest, &b);
}
/* net/recv! (net.clj:223-247): fills a 48-byte direct buffer (ms_msg) */
jint FN(recv)(JNIEnv* env, jclass c, jlong h, jint ep, jlong timeoutNs, jobject out) {
  (void)c;
  return ms_recv(H(h), (uint32_t)ep, timeoutNs, (ms_msg*)BUF(out));
}
/* the JSON envelope a node process prints / reads (process.clj:26-66,162) */
jlong FN(sendJson)(JNIEnv* env, jclass c, jlong h, jstring line) {
  (void)c;
  const char* s = (*env)->GetStringUTFChars(env, line, 0);
  const jlong rc = ms_send_json(H(h), s);
  (*env)->ReleaseStringUTFChars(env, line, s);
  return rc;
}
jint FN(recvJson)(JNIEnv* env, jclass c, jlong h, jint ep, jlong timeoutNs, jobject out, jlong cap) {
  (void)c;
  return ms_recv_json(H(h), (uint32_t)ep, timeoutNs, (char*)BUF(out), (size_t)cap);
}
/* closed-loop clients on the device: cfg = direct buffer holding an ms_gen_config; history records are ms_hist (32 B) */
jint FN(addGenClients)(JNIEnv* env, jclass c, jlong h, jobject cfg, jint firstName) {
  (void)c;
  return ms_add_gen_clients(H(h), (const ms_gen_config*)BUF(cfg), (uint32_t)firstName);
}
/* the lin-kv clients of the Raft nodes: cfg = direct buffer holding an ms_kv_gen_config */
jint FN(addKvClients)(JNIEnv* env, jclass c, jlong h, jobject cfg, jint firstName) {
  (void)c;
  return ms_add_kv_clients(H(h), (const ms_kv_gen_config*)BUF(cfg), (uint32_t)firstName);
}
jlong FN(historyDrain)(JNIEnv* env, jclass c, jlong h, jobject out, jlong cap) {
  (void)c;
  size_t n = 0;
  const int rc = ms_history_drain(H(h), (ms_hist*)BUF(out), (size_t)cap, &n);
  return rc < 0 ? (jlong)rc : (jlong)n;
}
/* the kafka clients of the single-node logs: cfg = direct buffer holding an ms_kafka_gen_config; records are
 * ms_kafka_hist (64 B) */
jint FN(addKafkaClients)(JNIEnv* env, jclass c, jlong h, jobject cfg, jint firstName) {
  (void)c;
  return ms_add_kafka_clients(H(h), (const ms_kafka_gen_config*)BUF(cfg), (uint32_t)firstName);
}
jlong FN(kafkaHistoryDrain)(JNIEnv* env, jclass c, jlong h, jobject out, jlong cap) {
  (void)c;
  size_t n = 0;
  const int rc = ms_kafka_history_drain(H(h), (ms_kafka_hist*)BUF(out), (size_t)cap, &n);
  return rc < 0 ? (jlong)rc : (jlong)n;
}
jint FN(addTxnRwClients)(JNIEnv* env, jclass c, jlong h, jobject cfg, jint firstName) {
  (void)c;
  return ms_add_txn_rw_clients(H(h), (const ms_txn_rw_gen_config*)BUF(cfg), (uint32_t)firstName);
}
jlong FN(txnRwHistoryDrain)(JNIEnv* env, jclass c, jlong h, jobject out, jlong cap) {
  (void)c;
  size_t n = 0;
  const int rc = ms_txn_rw_history_drain(H(h), (ms_txn_rw_hist*)BUF(out), (size_t)cap, &n);
  return rc < 0 ? (jlong)rc : (jlong)n;
}
jint FN(scheduleOps)(JNIEnv* env, jclass c, jlong h, jobject ops, jlong n) {
  (void)c;
  return ms_schedule_ops(H(h), (const ms_op*)BUF(ops), (size_t)n);
}

jint FN(step)(JNIEnv* env, jclass c, jlong h, jlong nRounds) { (void)env; (void)c; return ms_step(H(h), (uint64_t)nRounds); }
jint FN(run)(JNIEnv* env, jclass c, jlong h, jlong untilNs) { (void)env; (void)c; return ms_run(H(h), untilNs); }
jlong FN(now)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return ms_now(H(h)); }
jlong FN(round)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return (jlong)ms_round(H(h)); }
jint FN(setIdleJump)(JNIEnv* env, jclass c, jlong h, jint enable) { (void)env; (void)c; return ms_set_idle_jump(H(h), (int)enable); }

/* jepsen.net.proto/Net (net.clj:105-122) */
jint FN(netDrop)(JNIEnv* env, jclass c, jlong h, jint src, jint dest) { (void)env; (void)c; return ms_net_drop(H(h), (uint32_t)src, (uint32_t)dest); }
jint FN(netHeal)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return ms_net_heal(H(h)); }
jint FN(netSlow)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return ms_net_slow(H(h)); }
jint FN(netFast)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return ms_net_fast(H(h)); }
jint FN(netFlaky)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return ms_net_flaky(H(h)); }
jint FN(netSetLoss)(JNIEnv* env, jclass c, jlong h, jdouble p) { (void)env; (void)c; return ms_net_set_loss(H(h), p); }
jint FN(netPartition)(JNIEnv* env, jclass c, jlong h, jobject comp, jlong n) {
  (void)c;
  return ms_net_partition(H(h), (const uint32_t*)BUF(comp), (size_t)n);
}
/* partition nemesis: cfg = direct buffer holding an ms_nemesis_config; sides = direct buffer of g uint32 */
jint FN(setNemesis)(JNIEnv* env, jclass c, jlong h, jobject cfg) {
  (void)c;
  return ms_set_nemesis(H(h), (const ms_nemesis_config*)BUF(cfg));
}
jint FN(nemesisGrudge)(JNIEnv* env, jclass c, jint seedLo, jint seedHi, jint cluster, jint g, jint op, jint target,
                       jobject sides) {
  (void)c;
  return ms_nemesis_grudge((uint32_t)seedLo, (uint32_t)seedHi, (uint32_t)cluster, (uint32_t)g, (uint32_t)op,
                           (uint32_t)target, (uint32_t*)BUF(sides));
}

/* journal (net.clj:128-137, net/journal.clj:205-239) */
jint FN(journalOpen)(JNIEnv* env, jclass c, jlong h, jstring path) {
  (void)c;
  const char* s = (*env)->GetStringUTFChars(env, path, 0);
  const int rc = ms_journal_open(H(h), s);
  (*env)->ReleaseStringUTFChars(env, path, s);
  return rc;
}
jint FN(journalClose)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return ms_journal_close(H(h)); }
/* returns the number of events copied (>= 0) or an error code */
jlong FN(journalDrain)(JNIEnv* env, jclass c, jlong h, jobject events, jobject bodies, jlong cap) {
  (void)c;
  size_t n = 0;
  const int rc = ms_journal_drain(H(h), (ms_event*)BUF(events), (ms_jbody*)BUF(bodies), (size_t)cap, &n);
  return rc < 0 ? (jlong)rc : (jlong)n;
}
jlong FN(journalWritten)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return (jlong)ms_journal_written(H(h)); }

/* ms_run_streamed: the sink is a maelstrom.b200.Native$JournalSink; it is handed three direct
 * ByteBuffers (header, round rows, packed events) that are valid during the call only */
struct ms_jni_sink { JNIEnv* env; jobject sink; jmethodID accept; };
static int ms_jni_sink_call(void* ctx, const ms_jbatch* b, const ms_jround* rounds, const void* events) {
  struct ms_jni_sink* k = (struct ms_jni_sink*)ctx;
  JNIEnv* env = k->env;
  jobject jb = (*env)->NewDirectByteBuffer(env, (void*)b, (jlong)sizeof *b);
  jobject jr = (*env)->NewDirectByteBuffer(env, (void*)rounds, (jlong)(b->n_rounds * sizeof *rounds));
  jobject je = (*env)->NewDirectByteBuffer(env, (void*)events, (jlong)(b->n_events * b->format));
  const jint rc = (*env)->CallIntMethod(env, k->sink, k->accept, jb, jr, je);
  (*env)->DeleteLocalRef(env, jb); (*env)->DeleteLocalRef(env, jr); (*env)->DeleteLocalRef(env, je);
  return (*env)->ExceptionCheck(env) ? 1 : (int)rc;
}
jint FN(runStreamed)(JNIEnv* env, jclass c, jlong h, jlong untilNs, jint format, jlong bufEvents, jobject sink) {
  (void)c;
  struct ms_jni_sink k;
  k.env = env; k.sink = sink;
  k.accept = (*env)->GetMethodID(env, (*env)->GetObjectClass(env, sink), "accept",
                                 "(Ljava/nio/ByteBuffer;Ljava/nio/ByteBuffer;Ljava/nio/ByteBuffer;)I");
  if (!k.accept) return MS_ERR_ARG;
  return ms_run_streamed(H(h), untilNs, format, (size_t)bufEvents, ms_jni_sink_call, &k);
}
jint FN(journalDecode)(JNIEnv* env, jclass c, jobject batch, jobject rounds, jobject events, jobject out) {
  (void)c;
  return ms_journal_decode((const ms_jbatch*)BUF(batch), (const ms_jround*)BUF(rounds), BUF(events), (ms_event*)BUF(out));
}
/* MS_JFMT_4 batches are expanded by a decoder object that follows the stream */
jlong FN(jdecoderCreate)(JNIEnv* env, jclass c, jint log2Window) { (void)env; (void)c; return (jlong)(intptr_t)ms_jdecoder_create((uint32_t)log2Window); }
void FN(jdecoderDestroy)(JNIEnv* env, jclass c, jlong d) { (void)env; (void)c; ms_jdecoder_destroy((ms_jdecoder*)(intptr_t)d); }
jint FN(jdecoderDecode)(JNIEnv* env, jclass c, jlong d, jobject batch, jobject rounds, jobject events, jobject out) {
  (void)c;
  return ms_jdecoder_decode((ms_jdecoder*)(intptr_t)d, (const ms_jbatch*)BUF(batch), (const ms_jround*)BUF(rounds), BUF(events),
                            (ms_event*)BUF(out));
}
jint FN(jdecoderNote)(JNIEnv* env, jclass c, jlong d, jobject events, jlong n) {
  (void)c;
  return ms_jdecoder_note((ms_jdecoder*)(intptr_t)d, (const ms_event*)BUF(events), (size_t)n);
}
jstring FN(jdecoderError)(JNIEnv* env, jclass c, jlong d) { (void)c; return (*env)->NewStringUTF(env, ms_jdecoder_error((const ms_jdecoder*)(intptr_t)d)); }

/* read-backs: out = direct buffer of u64 */
jint FN(stats)(JNIEnv* env, jclass c, jlong h, jobject out9) { (void)c; return ms_stats(H(h), (uint64_t*)BUF(out9)); }
jlong FN(nodeSet)(JNIEnv* env, jclass c, jlong h, jint node, jobject values, jlong cap) {
  (void)c;
  return (jlong)ms_node_set(H(h), (uint32_t)node, (uint32_t*)BUF(values), (size_t)cap);
}
jlong FN(clientReplies)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return (jlong)ms_client_replies(H(h)); }
jlong FN(undeliverable)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return (jlong)ms_undeliverable(H(h)); }
jint FN(raftState)(JNIEnv* env, jclass c, jlong h, jint node, jobject out8) { (void)c; return ms_raft_state(H(h), (uint32_t)node, (uint64_t*)BUF(out8)); }
/* kafka read-backs: msgs = direct buffer of cap u32; returns the log's length or a negative error */
jlong FN(kafkaLog)(JNIEnv* env, jclass c, jlong h, jint node, jint key, jobject msgs, jlong cap) {
  (void)c;
  size_t n = 0;
  const int rc = ms_kafka_log(H(h), (uint32_t)node, (uint32_t)key, msgs ? (uint32_t*)BUF(msgs) : NULL, (size_t)cap, &n);
  return rc < 0 ? (jlong)rc : (jlong)n;
}
jlong FN(kafkaCommitted)(JNIEnv* env, jclass c, jlong h, jint node, jint key) { (void)env; (void)c; return ms_kafka_committed(H(h), (uint32_t)node, (uint32_t)key); }
/* the counter of a g-counter / pn-counter node: out = direct buffer of cap i64 (inc then dec); returns 2 x its block's
 * size or a negative error */
jint FN(counterState)(JNIEnv* env, jclass c, jlong h, jint node, jobject out, jlong cap) {
  (void)c;
  return ms_counter_state(H(h), (uint32_t)node, out ? (int64_t*)BUF(out) : NULL, (size_t)cap);
}
/* txn-rw-register read-backs: out = direct buffer of cap 40-B ms_txn_rw_entry; returns the log's length or a negative
 * error */
jint FN(txnRwLog)(JNIEnv* env, jclass c, jlong h, jint node, jobject out, jlong cap) {
  (void)c;
  return ms_txn_rw_log(H(h), (uint32_t)node, out ? (ms_txn_rw_entry*)BUF(out) : NULL, (size_t)cap);
}
/* lamport = direct buffer of one u64, logLen of one u32, values of cap u32, ts of cap u64; returns K or a negative error */
jint FN(txnRwState)(JNIEnv* env, jclass c, jlong h, jint node, jobject lamport, jobject logLen, jobject values, jobject ts,
                    jlong cap) {
  (void)c;
  return ms_txn_rw_state(H(h), (uint32_t)node, (uint64_t*)BUF(lamport), (uint32_t*)BUF(logLen), (uint32_t*)BUF(values),
                         (uint64_t*)BUF(ts), (size_t)cap);
}
jint FN(counters)(JNIEnv* env, jclass c, jlong h, jobject out8) { (void)c; return ms_counters(H(h), (uint64_t*)BUF(out8)); }
/* out = direct buffer of n u64 (>= 6 x n_nodes): tail / limit / head of the 48-B rings, then of the compact rings */
jint FN(ringCounters)(JNIEnv* env, jclass c, jlong h, jobject out, jint n) { (void)c; return ms_ring_counters(H(h), (uint64_t*)BUF(out), (uint32_t)n); }
/* test origin of a fresh simulation: round, message id, event id, ring counters ring_pos + e * ring_stride */
jint FN(setOrigin)(JNIEnv* env, jclass c, jlong h, jlong round, jlong msg_id, jlong event_id, jint ring_pos, jint ring_stride) {
  (void)env; (void)c;
  return ms_set_origin(H(h), (uint64_t)round, (uint64_t)msg_id, (uint64_t)event_id, (uint32_t)ring_pos, (uint32_t)ring_stride);
}

/* multi-GPU plumbing (one JVM per GPU, or one JVM driving several handles) */
jint FN(shardHandles)(JNIEnv* env, jclass c, jlong h, jobject blob) { (void)c; return ms_shard_handles(H(h), BUF(blob)); }
jint FN(shardConnect)(JNIEnv* env, jclass c, jlong h, jint peer, jobject blob) { (void)c; return ms_shard_connect(H(h), (uint32_t)peer, BUF(blob)); }
/* ms_set_barrier takes a C callback: only the built-in peer-memory barrier (fn = NULL) is reachable from the JVM */
jint FN(setBarrierDefault)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return ms_set_barrier(H(h), NULL, NULL); }
jlong FN(stream)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return (jlong)(intptr_t)ms_stream(H(h)); }
jint FN(shardOwner)(JNIEnv* env, jclass c, jint e, jint nServers, jint nShards) {
  (void)env; (void)c;
  return (jint)ms_shard_owner((uint32_t)e, (uint32_t)nServers, (uint32_t)nShards);
}

/* timing / diagnostics */
jint FN(timerBegin)(JNIEnv* env, jclass c, jlong h) { (void)env; (void)c; return ms_timer_begin(H(h)); }
jdouble FN(timerEnd)(JNIEnv* env, jclass c, jlong h) {
  (void)env; (void)c;
  double ms = 0;
  return ms_timer_end(H(h), &ms) < 0 ? -1.0 : ms;
}
jint FN(profile)(JNIEnv* env, jclass c, jlong h, jint enable) { (void)env; (void)c; return ms_profile(H(h), enable); }
/* out2 = direct buffer: f64 round-kernel ms, u64 launches */
jint FN(profileRead)(JNIEnv* env, jclass c, jlong h, jobject out2) {
  (void)c;
  unsigned char* o = (unsigned char*)BUF(out2);
  double ms = 0; uint64_t n = 0;
  const int rc = ms_profile_read(H(h), &ms, &n);
  memcpy(o, &ms, 8); memcpy(o + 8, &n, 8);
  return rc;
}
jint FN(debugPhaseCycles)(JNIEnv* env, jclass c, jlong h, jint enable, jobject out64) { (void)c; return ms_debug_phase_cycles(H(h), enable, (uint64_t*)BUF(out64)); }
jlong FN(topology)(JNIEnv* env, jclass c, jint topo, jint n, jint node, jobject out, jlong cap) {
  (void)c;
  return (jlong)ms_topology((uint32_t)topo, (uint32_t)n, (uint32_t)node, (uint32_t*)BUF(out), (size_t)cap);
}
#else
/* no <jni.h> on this box: the unit is intentionally empty */
typedef int ms_jni_translation_unit_is_empty_without_a_jdk;
#endif
