package akka.dispatch.verification

import java.nio.{ByteBuffer, ByteOrder}

/** The native half of the drop-in: one `@native` method per entry point of
  * include/demi_b200.h (bound by jni/DemiNative.c).  Not compiled in this
  * repository's image (no scalac); this is the binding a DEMi maintainer adds
  * next to `src/main/scala/verification/schedulers/`. */
object DemiNative {
  System.loadLibrary("demijni")
  @native def create(cfg: ByteBuffer): Long
  @native def destroy(h: Long): Unit
  @native def lastError(h: Long): String
  @native def setExternals(h: Long, events: ByteBuffer, n: Int): Int
  @native def fuzzBatch(h: Long, params: ByteBuffer, out: ByteBuffer): Int
  @native def fuzzTrace(h: Long, params: ByteBuffer, seed: Long, events: ByteBuffer, capEvents: Int,
                        depParent: ByteBuffer, capNodes: Int, counts: ByteBuffer, result: ByteBuffer): Int
  @native def setTrace(h: Long, events: ByteBuffer, nEvents: Int, externals: ByteBuffer, nExternals: Int): Int
  @native def replayBatch(h: Long, masks: ByteBuffer, nMasks: Int, maskWords: Int, lookingFor: Int, flags: Int,
                          out: ByteBuffer): Int
  @native def ddmin(h: Long, lookingFor: Int, flags: Int, checkUnmodified: Int, mcsMask: ByteBuffer, maskWords: Int,
                    iterationSizes: ByteBuffer, capIterations: Int, out: ByteBuffer): Int
  @native def stats(h: Long, out: ByteBuffer): Int
  @native def replayBatchEx(h: Long, masks: ByteBuffer, skipEvents: ByteBuffer, nTests: Int, maskWords: Int, lookingFor: Int,
                            flags: Int, out: ByteBuffer): Int
  @native def replayTrace(h: Long, mask: ByteBuffer, maskWords: Int, skipEvent: Int, lookingFor: Int, flags: Int,
                          events: ByteBuffer, capEvents: Int, count: ByteBuffer, result: ByteBuffer): Int
  @native def internalMinimize(h: Long, lookingFor: Int, flags: Int, events: ByteBuffer, capEvents: Int, sizes: ByteBuffer,
                               capSizes: Int, out: ByteBuffer): Int
  @native def setClockRules(h: Long, rules: ByteBuffer, nRules: Int, incrementTypes: ByteBuffer): Int
  @native def wildcardMinimize(h: Long, lookingFor: Int, flags: Int, events: ByteBuffer, capEvents: Int, sizes: ByteBuffer,
                               capSizes: Int, out: ByteBuffer): Int
  @native def dporBatch(h: Long, ext: ByteBuffer, extOffsets: ByteBuffer, nSearches: Int, params: ByteBuffer,
                        results: ByteBuffer, viol: ByteBuffer, capViol: Int): Int
  @native def dporBatchEx(h: Long, ext: ByteBuffer, extOffsets: ByteBuffer, nSearches: Int, params: ByteBuffer, flags: Int,
                          seedEvents: ByteBuffer, nSeedEvents: Int, seedParents: ByteBuffer, nSeedNodes: Int,
                          caps: ByteBuffer, capOffsets: ByteBuffer, results: ByteBuffer): Int
  @native def incrementalDdmin(h: Long, externals: ByteBuffer, nExternals: Int, params: ByteBuffer, flags: Int,
                               seedEvents: ByteBuffer, nSeedEvents: Int, seedParents: ByteBuffer, nSeedNodes: Int,
                               maxMaxDistance: Int, stopAtSize: Int, mcsMask: ByteBuffer, maskWords: Int, out: ByteBuffer): Int
  @native def provenance(h: Long, events: ByteBuffer, nEvents: Int, depParent: ByteBuffer, nNodes: Int, affectedMask: Int,
                         keepMask: ByteBuffer, maskWords: Int, out: ByteBuffer): Int
  @native def fuzzProvenance(h: Long, params: ByteBuffer, prefixIndex: ByteBuffer, n: Int, keepMasks: ByteBuffer,
                             maskWords: Int, out: ByteBuffer, results: ByteBuffer): Int
  @native def dedupCompact(h: Long, results: ByteBuffer, n: Long, mode: Int, outRecords: ByteBuffer, outIndex: ByteBuffer,
                           outCount: ByteBuffer): Int

  def direct(n: Int): ByteBuffer = ByteBuffer.allocateDirect(n).order(ByteOrder.LITTLE_ENDIAN)
  // ---- round 2
  /** demi_load_model: the data-only model of the application (include/demi_model_ir.h); `h` was created with model = 100. */
  @native def loadModel(h: Long, blob: ByteBuffer, size: Int): Int
  @native def actorIndex(h: Long, name: String): Int
  @native def actorName(h: Long, index: Int): String
  /** UnmodifiedEventDag.conjoinAtoms (minification/Util.scala:167-178) on the dag demi_ddmin minimizes. */
  @native def conjoinAtoms(h: Long, e1: Int, e2: Int): Int
  /** One DPORwHeuristics.test explored as a frontier of backtrack points (demi_frontier_params / demi_frontier_result). */
  @native def dporFrontier(h: Long, externals: ByteBuffer, n: Int, params: ByteBuffer, result: ByteBuffer,
                           viol: ByteBuffer, capViol: Int, hashes: ByteBuffer, capHashes: Long): Int
  /** All GPUs of the box from this JVM: n handles (jlongs in `handles`), NCCL wired up inside the library. */
  @native def createMulti(cfg: ByteBuffer, devices: ByteBuffer, n: Int, handles: ByteBuffer): Int
  @native def dporFrontierMulti(handles: ByteBuffer, n: Int, externals: ByteBuffer, nExt: Int, params: ByteBuffer,
                                results: ByteBuffer, viol: ByteBuffer, capViol: Int, hashes: ByteBuffer, capHashes: Long): Int
  @native def commUniqueId(id128: ByteBuffer): Int
  @native def commInit(h: Long, id128: ByteBuffer, rank: Int, world: Int): Int
  /** Fuzzer.generateFuzzTest, seeded (fuzzing/Fuzzer.scala:123-174). */
  @native def fuzzerGenerate(cfg: ByteBuffer, seed: Long, prefix: ByteBuffer, nPrefix: Int, postfix: ByteBuffer, nPostfix: Int,
                             out: ByteBuffer, cap: Int, nOut: ByteBuffer): Int
  /** demi_set_fuzzer / demi_fuzz_campaign: RunnerUtils.fuzz's loop (RunnerUtils.scala:75-91), a new program per execution */
  @native def setFuzzer(h: Long, cfg: ByteBuffer, prefix: ByteBuffer, nPrefix: Int, postfix: ByteBuffer, nPostfix: Int): Int
  @native def fuzzCampaign(h: Long, params: ByteBuffer, programSeedBase: Long, out: ByteBuffer): Int
  /** demi_random_ddmin: RunnerUtils.randomDDMin (RunnerUtils.scala:601-623), DDMin over RandomScheduler.test; params =
    * demi_fuzz_params with n_prefixes = max_executions.  iterationKeys: uint64 running sums of executions. */
  @native def randomDDMin(h: Long, params: ByteBuffer, checkUnmodified: Int, mcsMask: ByteBuffer, maskWords: Int,
                          iterationSizes: ByteBuffer, iterationKeys: ByteBuffer, cap: Int, out: ByteBuffer): Int
  /** demi_random_test_trace: the EventTrace RandomScheduler.test returns for a subsequence (the verified MCS trace) */
  @native def randomTestTrace(h: Long, mask: ByteBuffer, maskWords: Int, params: ByteBuffer, seed: Long, events: ByteBuffer,
                              capEvents: Int, count: ByteBuffer, result: ByteBuffer): Int
  /** demi_random_test_batch_many: test i is mask i over program traceOfTest(i) (offsets in elements), with that trace's
    * seedBase, maxMessages and lookingFor; the handle's program is not used */
  @native def randomTestBatchMany(h: Long, nTraces: Int, externals: ByteBuffer, extOffsets: ByteBuffer, nExternals: ByteBuffer,
                                  seedBase: ByteBuffer, maxMessages: ByteBuffer, lookingFor: ByteBuffer, traceOfTest: ByteBuffer,
                                  masks: ByteBuffer, nTests: Int, maskWords: Int, params: ByteBuffer, out: ByteBuffer): Int
  /** demi_random_ddmin_many: randomDDMin on every program t (its own seed, maxMessages = its trace's size, lookingFor),
    * every trace's tests in shared launches; status(t) is that trace's return code */
  @native def randomDDMinMany(h: Long, nTraces: Int, externals: ByteBuffer, extOffsets: ByteBuffer, nExternals: ByteBuffer,
                              seedBase: ByteBuffer, maxMessages: ByteBuffer, lookingFor: ByteBuffer, params: ByteBuffer,
                              checkUnmodified: Int, mcsMasks: ByteBuffer, maskWords: Int, iterationSizes: ByteBuffer,
                              iterationKeys: ByteBuffer, capIterations: Int, out: ByteBuffer, status: ByteBuffer): Int
  /** demi_fuzz_traces: the EventTraces of executions seed_base + prefixIndex(i), execution i at events + i*capEvents */
  @native def fuzzTraces(h: Long, params: ByteBuffer, prefixIndex: ByteBuffer, n: Int, events: ByteBuffer, capEvents: Int,
                         nEvents: ByteBuffer, results: ByteBuffer): Int
  /** demi_fuzz_traces_tree: fuzzTraces plus each execution's DepTracker tree, execution i's at depParent + i*capNodes */
  @native def fuzzTracesTree(h: Long, params: ByteBuffer, prefixIndex: ByteBuffer, n: Int, events: ByteBuffer, capEvents: Int,
                             nEvents: ByteBuffer, depParent: ByteBuffer, capNodes: Int, nNodes: ByteBuffer, results: ByteBuffer): Int
  /** demi_fuzz_traces_many: execution seeds(t) of program t (offsets in elements), or of the subsequence mask t keeps
    * (masks null: every event), with its own maxMessages and lookingFor, recorded in shared launches; depParent null: no
    * trees; status(t) is that trace's return code */
  @native def fuzzTracesMany(h: Long, nTraces: Int, externals: ByteBuffer, extOffsets: ByteBuffer, nExternals: ByteBuffer,
                             masks: ByteBuffer, maskWords: Int, seeds: ByteBuffer, maxMessages: ByteBuffer, lookingFor: ByteBuffer,
                             params: ByteBuffer, events: ByteBuffer, capEvents: Int, nEvents: ByteBuffer, depParent: ByteBuffer,
                             capNodes: Int, nNodes: ByteBuffer, results: ByteBuffer, status: ByteBuffer): Int
  /** demi_incremental_ddmin_many: RunnerUtils.editDistanceDporDDMin's minimisation of every trace t (offsets in elements;
    * seed t = seedEvents/seedParents at its offsets, seedEvents null: no seeds); status(t) is that trace's return code */
  @native def incrementalDdminMany(h: Long, nTraces: Int, externals: ByteBuffer, extOffsets: ByteBuffer, nExternals: ByteBuffer,
                                   seedEvents: ByteBuffer, seedEventOffsets: ByteBuffer, nSeedEvents: ByteBuffer,
                                   seedParents: ByteBuffer, seedParentOffsets: ByteBuffer, nSeedNodes: ByteBuffer,
                                   maxMessages: ByteBuffer, lookingFor: ByteBuffer, params: ByteBuffer, flags: Int,
                                   maxMaxDistance: Int, stopAtSize: Int, mcsMasks: ByteBuffer, maskWords: Int, out: ByteBuffer,
                                   status: ByteBuffer): Int
  /** demi_set_traces: a set of traces to minimise (offsets in elements), separate from setTrace's single trace */
  @native def setTraces(h: Long, nTraces: Int, events: ByteBuffer, eventOffsets: ByteBuffer, nEvents: ByteBuffer,
                        externals: ByteBuffer, extOffsets: ByteBuffer, nExternals: ByteBuffer): Int
  /** demi_replay_batch_many: test i replays mask i on trace traceOfTest(i); lookingFor holds one code per trace */
  @native def replayBatchMany(h: Long, traceOfTest: ByteBuffer, masks: ByteBuffer, nTests: Int, maskWords: Int,
                              lookingFor: ByteBuffer, flags: Int, out: ByteBuffer): Int
  /** demi_ddmin_many: RunnerUtils.stsSchedDDMin on every trace of the set; status(t) is that trace's return code */
  @native def ddminMany(h: Long, lookingFor: ByteBuffer, flags: Int, checkUnmodified: Int, mcsMasks: ByteBuffer, maskWords: Int,
                        iterationSizes: ByteBuffer, capIterations: Int, out: ByteBuffer, status: ByteBuffer): Int
  /** demi_replay_traces_many: test i replays mask i (null: full externals) on trace traceOfTest(i), leaving out trace event
   *  skipEvents(i) (null: none), and records its EventTrace at events + i*capEvents (verify_mcs's recording) */
  @native def replayTracesMany(h: Long, traceOfTest: ByteBuffer, masks: ByteBuffer, skipEvents: ByteBuffer, nTests: Int,
                               maskWords: Int, lookingFor: ByteBuffer, flags: Int, events: ByteBuffer, capEvents: Int,
                               nEvents: ByteBuffer, results: ByteBuffer): Int
  /** demi_internal_minimize_many: RunnerUtils.minimizeInternals on every trace of the set (verified MCS traces); trace t
   *  at traces + t*capEvents, status(t) its return code */
  @native def internalMinimizeMany(h: Long, lookingFor: ByteBuffer, flags: Int, traces: ByteBuffer, capEvents: Int,
                                   sizes: ByteBuffer, capSizes: Int, out: ByteBuffer, status: ByteBuffer): Int
  /** demi_wildcard_replay_batch_many: ClockClusterizer test i (an include mask over the deliveries of trace
   *  traceOfTest(i)) on that trace of the set */
  @native def wildcardReplayBatchMany(h: Long, traceOfTest: ByteBuffer, includeMasks: ByteBuffer, nTests: Int, maskWords: Int,
                                      lookingFor: ByteBuffer, flags: Int, out: ByteBuffer): Int
  /** demi_wildcard_minimize_many: WildcardMinimizer (STSSched, ClockClusterizer) on every trace of the set; trace t at
   *  traces + t*capEvents, status(t) its return code */
  @native def wildcardMinimizeMany(h: Long, lookingFor: ByteBuffer, flags: Int, traces: ByteBuffer, capEvents: Int,
                                   sizes: ByteBuffer, capSizes: Int, out: ByteBuffer, status: ByteBuffer): Int
  /** The flat experiment directory that replaces ExperimentSerializer's *.bin object streams (Serialization.scala:57-74). */
  @native def experimentSave(dir: String, exp: ByteBuffer): Int
  @native def experimentLoad(dir: String, exp: ByteBuffer): Int
  @native def addressOf(buf: ByteBuffer): Long

}

/** Flat encoding of the model-level vocabulary: an application registers, once,
  * how its actors and messages map to (actor index, type, p0, p1). */
trait ModelCodec {
  def model: Int                                   // DEMI_MODEL_*
  def modelFlags: Int
  def actorIndex(name: String): Int
  def encode(msg: Any): (Int, Int, Int)            // (type, p0, p1)  == the MessageFingerprint
  def violationCode(fp: ViolationFingerprint): Int
}

/** RandomScheduler whose explore() runs `max_executions` executions as ONE batch
  * on the GPU model and then confirms the first violating schedule on the real
  * application with ReplayScheduler (the reference's own validate_replay step,
  * RunnerUtils.scala:101-128). Signatures are unchanged. */
class GpuRandomScheduler(schedulerConfig: SchedulerConfig, codec: ModelCodec,
                         max_executions: Int = 1, invariant_check_interval: Int = 0, seed: Long = 0L)
    extends RandomScheduler(schedulerConfig, max_executions, invariant_check_interval,
                            new FullyRandom(seed = seed)) {
  private val cfg = DemiNative.direct(32)
  cfg.putInt(0, 0).putInt(4, codec.model).putInt(8, codec.modelFlags)
  private val h = DemiNative.create(cfg)
  require(h > 0, "demi_create failed: " + h)

  private def packExternals(trace: Seq[ExternalEvent]): ByteBuffer = {
    val b = DemiNative.direct(16 * trace.length)
    for ((e, i) <- trace.zipWithIndex) {
      val o = 16 * i
      e match {
        case s: Start => b.put(o, 1.toByte).put(o + 1, codec.actorIndex(s.name).toByte); b.putInt(o + 12, s._id)
        case k: Kill => b.put(o, 2.toByte).put(o + 1, codec.actorIndex(k.name).toByte); b.putInt(o + 12, k._id)
        case s: Send =>
          val (t, p0, p1) = codec.encode(s.messageCtor())
          b.put(o, 3.toByte).put(o + 1, codec.actorIndex(s.name).toByte).put(o + 3, t.toByte)
          b.putInt(o + 4, p0).putInt(o + 8, p1).putInt(o + 12, s._id)
        case w: WaitQuiescence => b.put(o, 4.toByte); b.putInt(o + 12, w._id)
        case p: Partition =>
          b.put(o, 5.toByte).put(o + 1, codec.actorIndex(p.a).toByte).put(o + 2, codec.actorIndex(p.b).toByte)
          b.putInt(o + 12, p._id)
        case u: UnPartition =>
          b.put(o, 6.toByte).put(o + 1, codec.actorIndex(u.a).toByte).put(o + 2, codec.actorIndex(u.b).toByte)
          b.putInt(o + 12, u._id)
        case other => throw new IllegalArgumentException("not representable in the data-only model: " + other)
      }
    }
    b
  }

  /** Seeds of all violating executions among seed .. seed + max_executions - 1. */
  def exploreBatch(trace: Seq[ExternalEvent], lookingFor: Option[ViolationFingerprint]): Seq[Long] = {
    if (test_invariant == null) throw new IllegalArgumentException("Must invoke setInvariant before test()")
    val rc = DemiNative.setExternals(h, packExternals(trace), trace.length)
    if (rc != 0) throw new IllegalArgumentException(DemiNative.lastError(h))
    val p = DemiNative.direct(32)
    p.putLong(0, seed).putLong(8, max_executions.toLong).putInt(16, if (maxMessages == Int.MaxValue) -1 else maxMessages)
    p.putInt(20, invariant_check_interval).putInt(24, lookingFor.map(codec.violationCode).getOrElse(0))
    val out = DemiNative.direct(32 * max_executions)
    val rc2 = DemiNative.fuzzBatch(h, p, out)
    if (rc2 != 0) throw new IllegalStateException(DemiNative.lastError(h))
    (0 until max_executions).filter(i => out.getInt(32 * i) != 0).map(i => seed + i)
  }
}
