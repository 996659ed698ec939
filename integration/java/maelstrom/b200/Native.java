package maelstrom.b200;

import java.nio.ByteBuffer;

/** Natives of maelstrom_b200/csrc/ms_jni.c: one per entry point of include/maelstrom_b200.h.
 *  Records cross as direct little-endian ByteBuffers in the C layout. */
public final class Native {
  static { System.loadLibrary("ms_jni"); }
  private Native() {}

  /** Receives one batch of the streamed journal (ms_run_streamed); buffers are valid during the call. */
  public interface JournalSink { int accept(ByteBuffer batch, ByteBuffer rounds, ByteBuffer events); }

  public static native int abiVersion();
  public static native long create(ByteBuffer msConfig);
  public static native void destroy(long h);
  public static native String lastError(long h);
  public static native int startNodes(long h, int workload);
  public static native int stopNodes(long h);
  public static native int addEndpoint(long h, String id, int kind);
  public static native int removeEndpoint(long h, int idx);
  public static native int endpointIndex(long h, String id);
  public static native long send(long h, int src, int dest, int type, int flags, int msgId, int inReplyTo, int p0, long p1);
  public static native int recv(long h, int endpoint, long timeoutNs, ByteBuffer msMsg48);
  public static native long sendJson(long h, String line);
  public static native int recvJson(long h, int endpoint, long timeoutNs, ByteBuffer outUtf8, long cap);
  public static native int addGenClients(long h, ByteBuffer msGenConfig, int firstName);
  public static native long historyDrain(long h, ByteBuffer msHist32, long cap);
  public static native int scheduleOps(long h, ByteBuffer msOps, long n);
  public static native int step(long h, long nRounds);
  public static native int run(long h, long untilNs);
  public static native long now(long h);
  public static native long round(long h);
  public static native int netDrop(long h, int src, int dest);
  public static native int netHeal(long h);
  public static native int netSlow(long h);
  public static native int netFast(long h);
  public static native int netFlaky(long h);
  public static native int netSetLoss(long h, double p);
  public static native int netPartition(long h, ByteBuffer componentIds, long n);
  public static native int journalOpen(long h, String path);
  public static native int journalClose(long h);
  public static native long journalDrain(long h, ByteBuffer events, ByteBuffer bodies, long cap);
  public static native long journalWritten(long h);
  public static native int runStreamed(long h, long untilNs, int format, long bufEvents, JournalSink sink);
  public static native int journalDecode(ByteBuffer batch, ByteBuffer rounds, ByteBuffer events, ByteBuffer outEvents);
  public static native long jdecoderCreate(int log2Window);
  public static native void jdecoderDestroy(long decoder);
  public static native int jdecoderDecode(long decoder, ByteBuffer batch, ByteBuffer rounds, ByteBuffer events, ByteBuffer outEvents);
  public static native int jdecoderNote(long decoder, ByteBuffer events, long n);
  public static native String jdecoderError(long decoder);
  public static native int stats(long h, ByteBuffer out9);
  public static native long nodeSet(long h, int node, ByteBuffer values, long cap);
  public static native long clientReplies(long h);
  public static native long undeliverable(long h);
  public static native int raftState(long h, int node, ByteBuffer out8);
  public static native int counters(long h, ByteBuffer out8);
  public static native int ringCounters(long h, ByteBuffer out, int n);
  public static native int setOrigin(long h, long round, long msgId, long eventId, int ringPos, int ringStride);
  public static native int shardHandles(long h, ByteBuffer blob512);
  public static native int shardConnect(long h, int peer, ByteBuffer blob512);
  public static native int setBarrierDefault(long h);
  public static native long stream(long h);
  public static native int shardOwner(int endpoint, int nServers, int nShards);
  public static native int timerBegin(long h);
  public static native double timerEnd(long h);
  public static native int profile(long h, int enable);
  public static native int profileRead(long h, ByteBuffer out2);
  public static native int debugPhaseCycles(long h, int enable, ByteBuffer out64);
  public static native long topology(int topology, int n, int node, ByteBuffer out, long cap);
}
