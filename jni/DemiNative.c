/*
 * JNI shim: one native method per C-ABI entry point of include/demi_b200.h.
 * Not compiled in this image (no JDK / jni.h); build on a JVM host with
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -I../include \
 *       DemiNative.c -L../demi_b200 -ldemi_b200 -o libdemijni.so
 * All buffers are direct java.nio.ByteBuffers (little-endian), so no copies
 * are made on the Java side; handles travel as jlong.
 * Scala side: jni/DemiNative.scala.
 */
#include <stdlib.h>
#include <jni.h>
#include <stdint.h>
#include "demi_b200.h"

#define H(h) ((demi_handle*)(intptr_t)(h))
#define BUF(env, b) ((*(env))->GetDirectBufferAddress((env), (b)))

JNIEXPORT jlong JNICALL Java_akka_dispatch_verification_DemiNative_create(JNIEnv* env, jclass c, jobject cfg) {
  demi_handle* h = 0;
  int32_t rc = demi_create((const demi_config*)BUF(env, cfg), &h);
  return rc == DEMI_OK ? (jlong)(intptr_t)h : (jlong)rc;          /* negative = error code */
}
JNIEXPORT void JNICALL Java_akka_dispatch_verification_DemiNative_destroy(JNIEnv* env, jclass c, jlong h) {
  demi_destroy(H(h));
}
JNIEXPORT jstring JNICALL Java_akka_dispatch_verification_DemiNative_lastError(JNIEnv* env, jclass c, jlong h) {
  return (*env)->NewStringUTF(env, demi_last_error(H(h)));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_setExternals(JNIEnv* env, jclass c, jlong h, jobject ev, jint n) {
  return demi_set_externals(H(h), (const demi_ext_event*)BUF(env, ev), (uint32_t)n);
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_fuzzBatch(JNIEnv* env, jclass c, jlong h, jobject params, jobject out) {
  return demi_fuzz_batch(H(h), (const demi_fuzz_params*)BUF(env, params), (demi_fuzz_result*)BUF(env, out));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_fuzzTrace(JNIEnv* env, jclass c, jlong h, jobject params, jlong seed,
    jobject events, jint capEvents, jobject depParent, jint capNodes, jobject counts /* 2 x u32 */, jobject result) {
  uint32_t* cnt = (uint32_t*)BUF(env, counts);
  return demi_fuzz_trace(H(h), (const demi_fuzz_params*)BUF(env, params), (int64_t)seed,
                         (demi_event*)BUF(env, events), (uint32_t)capEvents, &cnt[0],
                         (uint16_t*)BUF(env, depParent), (uint32_t)capNodes, &cnt[1],
                         (demi_fuzz_result*)BUF(env, result));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_setTrace(JNIEnv* env, jclass c, jlong h, jobject events, jint nEvents,
    jobject externals, jint nExternals) {
  return demi_set_trace(H(h), (const demi_event*)BUF(env, events), (uint32_t)nEvents,
                        (const demi_ext_event*)BUF(env, externals), (uint32_t)nExternals);
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_replayBatch(JNIEnv* env, jclass c, jlong h, jobject masks, jint nMasks,
    jint maskWords, jint lookingFor, jint flags, jobject out) {
  return demi_replay_batch(H(h), (const uint64_t*)BUF(env, masks), (uint32_t)nMasks, (uint32_t)maskWords,
                           (uint32_t)lookingFor, (uint32_t)flags, (demi_replay_result*)BUF(env, out));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_ddmin(JNIEnv* env, jclass c, jlong h, jint lookingFor, jint flags,
    jint checkUnmodified, jobject mcsMask, jint maskWords, jobject iterationSizes, jint capIterations, jobject out) {
  return demi_ddmin(H(h), (uint32_t)lookingFor, (uint32_t)flags, checkUnmodified, (uint64_t*)BUF(env, mcsMask),
                    (uint32_t)maskWords, (uint32_t*)BUF(env, iterationSizes), (uint32_t)capIterations,
                    (demi_ddmin_out*)BUF(env, out));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_stats(JNIEnv* env, jclass c, jlong h, jobject out) {
  return demi_stats(H(h), (demi_perf*)BUF(env, out));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_replayBatchEx(JNIEnv* env, jclass c, jlong h, jobject masks,
    jobject skipEvents, jint nTests, jint maskWords, jint lookingFor, jint flags, jobject out) {
  return demi_replay_batch_ex(H(h), masks ? (const uint64_t*)BUF(env, masks) : 0, skipEvents ? (const uint32_t*)BUF(env, skipEvents) : 0,
                              (uint32_t)nTests, (uint32_t)maskWords, (uint32_t)lookingFor, (uint32_t)flags,
                              (demi_replay_result*)BUF(env, out));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_replayTrace(JNIEnv* env, jclass c, jlong h, jobject mask, jint maskWords,
    jint skipEvent, jint lookingFor, jint flags, jobject events, jint capEvents, jobject count /* u32 */, jobject result) {
  return demi_replay_trace(H(h), (const uint64_t*)BUF(env, mask), (uint32_t)maskWords, (uint32_t)skipEvent, (uint32_t)lookingFor,
                           (uint32_t)flags, (demi_event*)BUF(env, events), (uint32_t)capEvents, (uint32_t*)BUF(env, count),
                           (demi_replay_result*)BUF(env, result));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_internalMinimize(JNIEnv* env, jclass c, jlong h, jint lookingFor,
    jint flags, jobject events, jint capEvents, jobject sizes, jint capSizes, jobject out) {
  return demi_internal_minimize(H(h), (uint32_t)lookingFor, (uint32_t)flags, (demi_event*)BUF(env, events), (uint32_t)capEvents,
                                (uint32_t*)BUF(env, sizes), (uint32_t)capSizes, (demi_intmin_out*)BUF(env, out));
}
/* rules: nRules packed u32 (DEMI_CLOCK_RULE); incrementTypes: 8 u32 words, may be null */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_setClockRules(JNIEnv* env, jclass c, jlong h, jobject rules,
    jint nRules, jobject incrementTypes) {
  return demi_set_clock_rules(H(h), rules ? (const uint32_t*)BUF(env, rules) : 0, (uint32_t)nRules,
                              incrementTypes ? (const uint32_t*)BUF(env, incrementTypes) : 0);
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_wildcardMinimize(JNIEnv* env, jclass c, jlong h, jint lookingFor,
    jint flags, jobject events, jint capEvents, jobject sizes, jint capSizes, jobject out) {
  return demi_wildcard_minimize(H(h), (uint32_t)lookingFor, (uint32_t)flags, (demi_event*)BUF(env, events), (uint32_t)capEvents,
                                (uint32_t*)BUF(env, sizes), (uint32_t)capSizes, (demi_intmin_out*)BUF(env, out));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_dporBatch(JNIEnv* env, jclass c, jlong h, jobject ext, jobject extOffsets,
    jint nSearches, jobject params, jobject results, jobject viol, jint capViol) {
  return demi_dpor_batch(H(h), (const demi_ext_event*)BUF(env, ext), (const uint32_t*)BUF(env, extOffsets), (uint32_t)nSearches,
                         (const demi_dpor_params*)BUF(env, params), (demi_dpor_result*)BUF(env, results),
                         viol ? (demi_dpor_violation*)BUF(env, viol) : 0, (uint32_t)capViol, 0, 0);
}
/* seed = {events, nEvents, depParent, nNodes}; caps / capOffsets may be null (one uncapped test per instance) */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_dporBatchEx(JNIEnv* env, jclass c, jlong h, jobject ext, jobject extOffsets,
    jint nSearches, jobject params, jint flags, jobject seedEvents, jint nSeedEvents, jobject seedParents, jint nSeedNodes,
    jobject caps, jobject capOffsets, jobject results) {
  demi_dpor_seed seed = { seedEvents ? (const demi_event*)BUF(env, seedEvents) : 0, (uint32_t)nSeedEvents,
                          seedParents ? (const uint16_t*)BUF(env, seedParents) : 0, (uint32_t)nSeedNodes };
  demi_dpor_ex ex = { (uint32_t)flags, seedEvents ? &seed : 0, caps ? (const int32_t*)BUF(env, caps) : 0,
                      capOffsets ? (const uint32_t*)BUF(env, capOffsets) : 0 };
  return demi_dpor_batch_ex(H(h), (const demi_ext_event*)BUF(env, ext), (const uint32_t*)BUF(env, extOffsets), (uint32_t)nSearches,
                            (const demi_dpor_params*)BUF(env, params), &ex, (demi_dpor_result*)BUF(env, results), 0, 0, 0, 0);
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_incrementalDdmin(JNIEnv* env, jclass c, jlong h, jobject externals,
    jint nExternals, jobject params, jint flags, jobject seedEvents, jint nSeedEvents, jobject seedParents, jint nSeedNodes,
    jint maxMaxDistance, jint stopAtSize, jobject mcsMask, jint maskWords, jobject out) {
  demi_dpor_seed seed = { (const demi_event*)BUF(env, seedEvents), (uint32_t)nSeedEvents,
                          (const uint16_t*)BUF(env, seedParents), (uint32_t)nSeedNodes };
  return demi_incremental_ddmin(H(h), (const demi_ext_event*)BUF(env, externals), (uint32_t)nExternals,
                                (const demi_dpor_params*)BUF(env, params), (uint32_t)flags, &seed, maxMaxDistance,
                                (uint32_t)stopAtSize, (uint64_t*)BUF(env, mcsMask), (uint32_t)maskWords,
                                (demi_incddmin_out*)BUF(env, out));
}
/* demi_incremental_ddmin_many: seed t's events are seedEvents[seedEventOffsets[t] ..] (nSeedEvents[t] records) and its
 * DepTracker tree seedParents[seedParentOffsets[t] ..] (nSeedNodes[t] entries); seedEvents null: no trace has a seed */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_incrementalDdminMany(JNIEnv* env, jclass c, jlong h, jint nTraces,
    jobject externals, jobject extOffsets, jobject nExternals, jobject seedEvents, jobject seedEventOffsets, jobject nSeedEvents,
    jobject seedParents, jobject seedParentOffsets, jobject nSeedNodes, jobject maxMessages, jobject lookingFor, jobject params,
    jint flags, jint maxMaxDistance, jint stopAtSize, jobject mcsMasks, jint maskWords, jobject out, jobject status) {
  demi_dpor_seed* seeds = 0;
  if (seedEvents && nTraces > 0) {
    const demi_event* ev = (const demi_event*)BUF(env, seedEvents);
    const uint16_t* par = (const uint16_t*)BUF(env, seedParents);
    const uint32_t* eo = (const uint32_t*)BUF(env, seedEventOffsets); const uint32_t* ne = (const uint32_t*)BUF(env, nSeedEvents);
    const uint32_t* po = (const uint32_t*)BUF(env, seedParentOffsets); const uint32_t* nn = (const uint32_t*)BUF(env, nSeedNodes);
    seeds = (demi_dpor_seed*)malloc((size_t)nTraces * sizeof(demi_dpor_seed));
    if (!seeds) return DEMI_ERR_CAPACITY;
    for (jint t = 0; t < nTraces; t++) {
      seeds[t].events = ev + eo[t]; seeds[t].n_events = ne[t];
      seeds[t].dep_parent = par + po[t]; seeds[t].n_nodes = nn[t];
    }
  }
  const int32_t rc = demi_incremental_ddmin_many(H(h), (uint32_t)nTraces, (const demi_ext_event*)BUF(env, externals),
                                                 (const uint32_t*)BUF(env, extOffsets), (const uint32_t*)BUF(env, nExternals), seeds,
                                                 (const int32_t*)BUF(env, maxMessages), (const uint32_t*)BUF(env, lookingFor),
                                                 (const demi_dpor_params*)BUF(env, params), (uint32_t)flags, maxMaxDistance,
                                                 (uint32_t)stopAtSize, (uint64_t*)BUF(env, mcsMasks), (uint32_t)maskWords,
                                                 (demi_incddmin_out*)BUF(env, out), (int32_t*)BUF(env, status));
  free(seeds);
  return rc;
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_provenance(JNIEnv* env, jclass c, jlong h, jobject events, jint nEvents,
    jobject depParent, jint nNodes, jint affectedMask, jobject keepMask, jint maskWords, jobject out) {
  return demi_provenance(H(h), (const demi_event*)BUF(env, events), (uint32_t)nEvents, (const uint16_t*)BUF(env, depParent),
                         (uint32_t)nNodes, (uint32_t)affectedMask, (uint64_t*)BUF(env, keepMask), (uint32_t)maskWords,
                         (demi_provenance_out*)BUF(env, out));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_fuzzProvenance(JNIEnv* env, jclass c, jlong h, jobject params,
    jobject prefixIndex, jint n, jobject keepMasks, jint maskWords, jobject out, jobject results) {
  return demi_fuzz_provenance(H(h), (const demi_fuzz_params*)BUF(env, params), (const uint32_t*)BUF(env, prefixIndex), (uint32_t)n,
                              (uint64_t*)BUF(env, keepMasks), (uint32_t)maskWords, (demi_provenance_out*)BUF(env, out),
                              results ? (demi_fuzz_result*)BUF(env, results) : 0);
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_dedupCompact(JNIEnv* env, jclass c, jlong h, jobject results, jlong n,
    jint mode, jobject outRecords, jobject outIndex, jobject outCount /* u64 */) {
  return demi_dedup_compact(H(h), (const demi_fuzz_result*)BUF(env, results), (uint64_t)n, mode,
                            (demi_fuzz_result*)BUF(env, outRecords), outIndex ? (uint32_t*)BUF(env, outIndex) : 0,
                            (uint64_t*)BUF(env, outCount));
}

/* ---- round 2: loaded models, frontier DPOR on one or several GPUs, conjoined atoms, fuzzer, experiment directory */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_loadModel(JNIEnv* env, jclass c, jlong h, jobject blob, jint size) {
  return demi_load_model(H(h), BUF(env, blob), (size_t)size);
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_actorIndex(JNIEnv* env, jclass c, jlong h, jstring name) {
  const char* s = (*env)->GetStringUTFChars(env, name, 0);
  jint r = demi_actor_index(H(h), s);
  (*env)->ReleaseStringUTFChars(env, name, s);
  return r;
}
JNIEXPORT jstring JNICALL Java_akka_dispatch_verification_DemiNative_actorName(JNIEnv* env, jclass c, jlong h, jint index) {
  const char* s = demi_actor_name(H(h), (uint32_t)index);
  return s ? (*env)->NewStringUTF(env, s) : 0;
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_conjoinAtoms(JNIEnv* env, jclass c, jlong h, jint e1, jint e2) {
  return demi_conjoin_atoms(H(h), (uint32_t)e1, (uint32_t)e2);
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_dporFrontier(JNIEnv* env, jclass c, jlong h, jobject externals, jint n,
    jobject params, jobject result, jobject viol, jint capViol, jobject hashes, jlong capHashes) {
  return demi_dpor_frontier(H(h), (const demi_ext_event*)BUF(env, externals), (uint32_t)n, (const demi_frontier_params*)BUF(env, params),
                            (demi_frontier_result*)BUF(env, result), viol ? (demi_dpor_violation*)BUF(env, viol) : 0, (uint32_t)capViol,
                            hashes ? (uint64_t*)BUF(env, hashes) : 0, (uint64_t)capHashes);
}
/* one JVM process drives all the GPUs of the box: handles[] is a direct buffer of n jlongs */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_createMulti(JNIEnv* env, jclass c, jobject cfg, jobject devices, jint n,
    jobject handles) {
  return demi_create_multi((const demi_config*)BUF(env, cfg), (const int32_t*)BUF(env, devices), n, (demi_handle**)BUF(env, handles));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_dporFrontierMulti(JNIEnv* env, jclass c, jobject handles, jint n,
    jobject externals, jint nExt, jobject params, jobject results, jobject viol, jint capViol, jobject hashes, jlong capHashes) {
  return demi_dpor_frontier_multi((demi_handle**)BUF(env, handles), n, (const demi_ext_event*)BUF(env, externals), (uint32_t)nExt,
                                  (const demi_frontier_params*)BUF(env, params), (demi_frontier_result*)BUF(env, results),
                                  viol ? (demi_dpor_violation*)BUF(env, viol) : 0, (uint32_t)capViol,
                                  hashes ? (uint64_t*)BUF(env, hashes) : 0, (uint64_t)capHashes);
}
/* one process per GPU (e.g. one JVM per device): rank 0 makes the id, the host ships its 128 bytes, every rank joins */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_commUniqueId(JNIEnv* env, jclass c, jobject id128) {
  return demi_comm_unique_id((uint8_t*)BUF(env, id128));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_commInit(JNIEnv* env, jclass c, jlong h, jobject id128, jint rank, jint world) {
  return demi_comm_init(H(h), (const uint8_t*)BUF(env, id128), rank, world);
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_fuzzerGenerate(JNIEnv* env, jclass c, jobject cfg, jlong seed,
    jobject prefix, jint nPrefix, jobject postfix, jint nPostfix, jobject out, jint cap, jobject nOut /* u32 */) {
  return demi_fuzzer_generate((const demi_fuzzer_config*)BUF(env, cfg), (int64_t)seed, (const demi_ext_event*)BUF(env, prefix), (uint32_t)nPrefix,
                              postfix ? (const demi_ext_event*)BUF(env, postfix) : 0, (uint32_t)nPostfix, (demi_ext_event*)BUF(env, out),
                              (uint32_t)cap, (uint32_t*)BUF(env, nOut));
}
/* demi_set_fuzzer / demi_fuzz_campaign: RunnerUtils.fuzz's loop with a new Fuzzer program per execution */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_setFuzzer(JNIEnv* env, jclass c, jlong h, jobject cfg,
    jobject prefix, jint nPrefix, jobject postfix, jint nPostfix) {
  return demi_set_fuzzer(H(h), (const demi_fuzzer_config*)BUF(env, cfg), (const demi_ext_event*)BUF(env, prefix), (uint32_t)nPrefix,
                         postfix ? (const demi_ext_event*)BUF(env, postfix) : 0, (uint32_t)nPostfix);
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_fuzzCampaign(JNIEnv* env, jclass c, jlong h, jobject params,
    jlong programSeedBase, jobject out) {
  return demi_fuzz_campaign(H(h), (const demi_fuzz_params*)BUF(env, params), (int64_t)programSeedBase, (demi_fuzz_result*)BUF(env, out));
}
/* demi_random_ddmin / demi_random_test_trace: RunnerUtils.randomDDMin, DDMin with a RandomScheduler as the TestOracle,
 * over the program of setExternals (the verified trace: randomTestTrace on the MCS mask at seed + mcs_first_hit) */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_randomDDMin(JNIEnv* env, jclass c, jlong h, jobject params,
    jint checkUnmodified, jobject mcsMask, jint maskWords, jobject iterationSizes, jobject iterationKeys, jint cap, jobject out) {
  return demi_random_ddmin(H(h), (const demi_fuzz_params*)BUF(env, params), checkUnmodified, (uint64_t*)BUF(env, mcsMask),
                           (uint32_t)maskWords, iterationSizes ? (uint32_t*)BUF(env, iterationSizes) : 0,
                           iterationKeys ? (uint64_t*)BUF(env, iterationKeys) : 0, (uint32_t)cap, (demi_random_ddmin_out*)BUF(env, out));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_randomTestTrace(JNIEnv* env, jclass c, jlong h, jobject mask,
    jint maskWords, jobject params, jlong seed, jobject events, jint capEvents, jobject count, jobject result) {
  return demi_random_test_trace(H(h), (const uint64_t*)BUF(env, mask), (uint32_t)maskWords, (const demi_fuzz_params*)BUF(env, params),
                                (int64_t)seed, (demi_event*)BUF(env, events), (uint32_t)capEvents, (uint32_t*)BUF(env, count),
                                (demi_fuzz_result*)BUF(env, result));
}
/* demi_random_test_batch_many / demi_random_ddmin_many: the same over many programs (offsets in elements), each with its
 * own seed base, max_messages and looking_for; status[t] is trace t's return code */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_randomTestBatchMany(JNIEnv* env, jclass c, jlong h, jint nTraces,
    jobject externals, jobject extOffsets, jobject nExternals, jobject seedBase, jobject maxMessages, jobject lookingFor,
    jobject traceOfTest, jobject masks, jint nTests, jint maskWords, jobject params, jobject out) {
  return demi_random_test_batch_many(H(h), (uint32_t)nTraces, (const demi_ext_event*)BUF(env, externals),
                                     (const uint32_t*)BUF(env, extOffsets), (const uint32_t*)BUF(env, nExternals),
                                     (const int64_t*)BUF(env, seedBase), (const int32_t*)BUF(env, maxMessages),
                                     (const uint32_t*)BUF(env, lookingFor), (const uint32_t*)BUF(env, traceOfTest),
                                     (const uint64_t*)BUF(env, masks), (uint32_t)nTests, (uint32_t)maskWords,
                                     (const demi_fuzz_params*)BUF(env, params), (demi_random_test_result*)BUF(env, out));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_randomDDMinMany(JNIEnv* env, jclass c, jlong h, jint nTraces,
    jobject externals, jobject extOffsets, jobject nExternals, jobject seedBase, jobject maxMessages, jobject lookingFor,
    jobject params, jint checkUnmodified, jobject mcsMasks, jint maskWords, jobject iterationSizes, jobject iterationKeys,
    jint capIterations, jobject out, jobject status) {
  return demi_random_ddmin_many(H(h), (uint32_t)nTraces, (const demi_ext_event*)BUF(env, externals),
                                (const uint32_t*)BUF(env, extOffsets), (const uint32_t*)BUF(env, nExternals),
                                (const int64_t*)BUF(env, seedBase), (const int32_t*)BUF(env, maxMessages),
                                (const uint32_t*)BUF(env, lookingFor), (const demi_fuzz_params*)BUF(env, params), checkUnmodified,
                                (uint64_t*)BUF(env, mcsMasks), (uint32_t)maskWords,
                                iterationSizes ? (uint32_t*)BUF(env, iterationSizes) : 0,
                                iterationKeys ? (uint64_t*)BUF(env, iterationKeys) : 0, (uint32_t)capIterations,
                                (demi_random_ddmin_out*)BUF(env, out), (int32_t*)BUF(env, status));
}
/* demi_fuzz_traces / demi_set_traces / demi_replay_batch_many / demi_ddmin_many: many violating executions recorded,
 * replayed and minimized with their tests in shared launches */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_fuzzTraces(JNIEnv* env, jclass c, jlong h, jobject params,
    jobject prefixIndex, jint n, jobject events, jint capEvents, jobject nEvents, jobject results) {
  return demi_fuzz_traces(H(h), (const demi_fuzz_params*)BUF(env, params), (const uint32_t*)BUF(env, prefixIndex), (uint32_t)n,
                          (demi_event*)BUF(env, events), (uint32_t)capEvents, (uint32_t*)BUF(env, nEvents),
                          results ? (demi_fuzz_result*)BUF(env, results) : 0);
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_fuzzTracesTree(JNIEnv* env, jclass c, jlong h, jobject params,
    jobject prefixIndex, jint n, jobject events, jint capEvents, jobject nEvents, jobject depParent, jint capNodes, jobject nNodes,
    jobject results) {
  return demi_fuzz_traces_tree(H(h), (const demi_fuzz_params*)BUF(env, params), (const uint32_t*)BUF(env, prefixIndex), (uint32_t)n,
                               (demi_event*)BUF(env, events), (uint32_t)capEvents, (uint32_t*)BUF(env, nEvents),
                               (uint16_t*)BUF(env, depParent), (uint32_t)capNodes, (uint32_t*)BUF(env, nNodes),
                               results ? (demi_fuzz_result*)BUF(env, results) : 0);
}
/* demi_fuzz_traces_many: execution seeds[t] of program t (offsets in elements), or of the subsequence mask t keeps (masks
 * null: every event), each with its own maxMessages and lookingFor; status[t] is trace t's return code */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_fuzzTracesMany(JNIEnv* env, jclass c, jlong h, jint nTraces,
    jobject externals, jobject extOffsets, jobject nExternals, jobject masks, jint maskWords, jobject seeds, jobject maxMessages,
    jobject lookingFor, jobject params, jobject events, jint capEvents, jobject nEvents, jobject depParent, jint capNodes,
    jobject nNodes, jobject results, jobject status) {
  return demi_fuzz_traces_many(H(h), (uint32_t)nTraces, (const demi_ext_event*)BUF(env, externals),
                               (const uint32_t*)BUF(env, extOffsets), (const uint32_t*)BUF(env, nExternals),
                               masks ? (const uint64_t*)BUF(env, masks) : 0, (uint32_t)maskWords, (const int64_t*)BUF(env, seeds),
                               (const int32_t*)BUF(env, maxMessages), (const uint32_t*)BUF(env, lookingFor),
                               (const demi_fuzz_params*)BUF(env, params), (demi_event*)BUF(env, events), (uint32_t)capEvents,
                               (uint32_t*)BUF(env, nEvents), depParent ? (uint16_t*)BUF(env, depParent) : 0, (uint32_t)capNodes,
                               nNodes ? (uint32_t*)BUF(env, nNodes) : 0, results ? (demi_fuzz_result*)BUF(env, results) : 0,
                               (int32_t*)BUF(env, status));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_setTraces(JNIEnv* env, jclass c, jlong h, jint nTraces,
    jobject events, jobject eventOffsets, jobject nEvents, jobject externals, jobject extOffsets, jobject nExternals) {
  return demi_set_traces(H(h), (uint32_t)nTraces, (const demi_event*)BUF(env, events), (const uint32_t*)BUF(env, eventOffsets),
                         (const uint32_t*)BUF(env, nEvents), (const demi_ext_event*)BUF(env, externals),
                         (const uint32_t*)BUF(env, extOffsets), (const uint32_t*)BUF(env, nExternals));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_replayBatchMany(JNIEnv* env, jclass c, jlong h, jobject traceOfTest,
    jobject masks, jint nTests, jint maskWords, jobject lookingFor, jint flags, jobject out) {
  return demi_replay_batch_many(H(h), (const uint32_t*)BUF(env, traceOfTest), (const uint64_t*)BUF(env, masks), (uint32_t)nTests,
                                (uint32_t)maskWords, (const uint32_t*)BUF(env, lookingFor), (uint32_t)flags,
                                (demi_replay_result*)BUF(env, out));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_ddminMany(JNIEnv* env, jclass c, jlong h, jobject lookingFor,
    jint flags, jint checkUnmodified, jobject mcsMasks, jint maskWords, jobject iterationSizes, jint capIterations, jobject out,
    jobject status) {
  return demi_ddmin_many(H(h), (const uint32_t*)BUF(env, lookingFor), (uint32_t)flags, checkUnmodified, (uint64_t*)BUF(env, mcsMasks),
                         (uint32_t)maskWords, iterationSizes ? (uint32_t*)BUF(env, iterationSizes) : 0, (uint32_t)capIterations,
                         (demi_ddmin_out*)BUF(env, out), (int32_t*)BUF(env, status));
}
/* demi_replay_traces_many / demi_internal_minimize_many: the verified MCS traces of the set recorded, and their internal
 * events minimized, with their tests in shared launches */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_replayTracesMany(JNIEnv* env, jclass c, jlong h, jobject traceOfTest,
    jobject masks, jobject skipEvents, jint nTests, jint maskWords, jobject lookingFor, jint flags, jobject events, jint capEvents,
    jobject nEvents, jobject results) {
  return demi_replay_traces_many(H(h), (const uint32_t*)BUF(env, traceOfTest), masks ? (const uint64_t*)BUF(env, masks) : 0,
                                 skipEvents ? (const uint32_t*)BUF(env, skipEvents) : 0, (uint32_t)nTests, (uint32_t)maskWords,
                                 (const uint32_t*)BUF(env, lookingFor), (uint32_t)flags, (demi_event*)BUF(env, events),
                                 (uint32_t)capEvents, (uint32_t*)BUF(env, nEvents), (demi_replay_result*)BUF(env, results));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_internalMinimizeMany(JNIEnv* env, jclass c, jlong h,
    jobject lookingFor, jint flags, jobject traces, jint capEvents, jobject sizes, jint capSizes, jobject out, jobject status) {
  return demi_internal_minimize_many(H(h), (const uint32_t*)BUF(env, lookingFor), (uint32_t)flags, (demi_event*)BUF(env, traces),
                                     (uint32_t)capEvents, sizes ? (uint32_t*)BUF(env, sizes) : 0, (uint32_t)capSizes,
                                     (demi_intmin_out*)BUF(env, out), (int32_t*)BUF(env, status));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_wildcardReplayBatchMany(JNIEnv* env, jclass c, jlong h,
    jobject traceOfTest, jobject includeMasks, jint nTests, jint maskWords, jobject lookingFor, jint flags, jobject out) {
  return demi_wildcard_replay_batch_many(H(h), (const uint32_t*)BUF(env, traceOfTest), (const uint64_t*)BUF(env, includeMasks),
                                         (uint32_t)nTests, (uint32_t)maskWords, (const uint32_t*)BUF(env, lookingFor),
                                         (uint32_t)flags, (demi_replay_result*)BUF(env, out));
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_wildcardMinimizeMany(JNIEnv* env, jclass c, jlong h,
    jobject lookingFor, jint flags, jobject traces, jint capEvents, jobject sizes, jint capSizes, jobject out, jobject status) {
  return demi_wildcard_minimize_many(H(h), (const uint32_t*)BUF(env, lookingFor), (uint32_t)flags, (demi_event*)BUF(env, traces),
                                     (uint32_t)capEvents, sizes ? (uint32_t*)BUF(env, sizes) : 0, (uint32_t)capSizes,
                                     (demi_intmin_out*)BUF(env, out), (int32_t*)BUF(env, status));
}
/* `exp` = a direct buffer laid out as demi_experiment whose pointer fields the Scala side fills with
 * GetDirectBufferAddress-style addresses (DemiNative.addressOf) */
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_experimentSave(JNIEnv* env, jclass c, jstring dir, jobject exp) {
  const char* s = (*env)->GetStringUTFChars(env, dir, 0);
  jint r = demi_experiment_save(s, (const demi_experiment*)BUF(env, exp));
  (*env)->ReleaseStringUTFChars(env, dir, s);
  return r;
}
JNIEXPORT jint JNICALL Java_akka_dispatch_verification_DemiNative_experimentLoad(JNIEnv* env, jclass c, jstring dir, jobject exp) {
  const char* s = (*env)->GetStringUTFChars(env, dir, 0);
  jint r = demi_experiment_load(s, (demi_experiment*)BUF(env, exp));
  (*env)->ReleaseStringUTFChars(env, dir, s);
  return r;
}
JNIEXPORT jlong JNICALL Java_akka_dispatch_verification_DemiNative_addressOf(JNIEnv* env, jclass c, jobject buf) {
  return (jlong)(intptr_t)BUF(env, buf);
}
