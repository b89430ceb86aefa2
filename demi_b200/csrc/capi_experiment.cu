// capi_experiment.cu — host-only entry points of the C ABI: the seeded Fuzzer (fuzzing/Fuzzer.scala:24-194) and the
// flat experiment directory that replaces the reference's Java-serialized *.bin files (Serialization.scala:57-74,
// :176-254).  No device code; lives in the library so that a JVM host gets them through the same JNI shim.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include <sys/stat.h>
#include "engine.hpp"
#include "fuzzer_gen.cuh"

// Fuzzer.generateFuzzTest (Fuzzer.scala:123-174): the body is fuzzer_gen.cuh, shared with the campaign's generator kernel.
extern "C" int32_t demi_fuzzer_generate(const demi_fuzzer_config* cfg, int64_t seed,
                                        const demi_ext_event* prefix, uint32_t n_prefix,
                                        const demi_ext_event* postfix, uint32_t n_postfix,
                                        demi_ext_event* out, uint32_t cap, uint32_t* n_out) {
  if (!cfg || !out || !n_out || (!prefix && n_prefix) || (!postfix && n_postfix))
    return fail(nullptr, DEMI_ERR_INVALID, "demi_fuzzer_generate: null argument");
  uint32_t starts = 0;
  for (uint32_t i = 0; i < n_prefix; i++) starts += prefix[i].kind == DEMI_EXT_START;
  std::vector<uint8_t> alive(std::max(starts, 1u));
  std::vector<uint16_t> pairs(2 * (size_t)demi::fuzzer_pair_room(starts) + 1);
  std::vector<demi_ext_event> test((size_t)demi::fuzzer_program_room(*cfg, n_prefix, n_postfix));
  uint32_t sends = 0;
  const uint32_t len = demi::fuzzer_generate(*cfg, seed, prefix, n_prefix, postfix, n_postfix, alive.data(), pairs.data(),
                                             test.data(), &sends);
  *n_out = len;
  if (len > cap) return fail(nullptr, DEMI_ERR_CAPACITY, "demi_fuzzer_generate: %u events, room for %u", len, cap);
  std::copy(test.begin(), test.begin() + len, out);
  return DEMI_OK;
}

// ---- flat experiment directory: raw little-endian arrays of the C-ABI records + meta.json
namespace {
bool write_file(const std::string& p, const void* data, size_t bytes) {
  FILE* f = fopen(p.c_str(), "wb"); if (!f) return false;
  const bool ok = !bytes || fwrite(data, 1, bytes, f) == bytes;
  return fclose(f) == 0 && ok;
}
long file_size(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0 ? (long)st.st_size : -1; }
bool read_file(const std::string& p, void* data, size_t bytes) {
  FILE* f = fopen(p.c_str(), "rb"); if (!f) return false;
  const bool ok = !bytes || fread(data, 1, bytes, f) == bytes;
  fclose(f); return ok;
}
long json_int(const std::string& txt, const char* key, long dflt) {
  const std::string k = std::string("\"") + key + "\"";
  size_t p = txt.find(k); if (p == std::string::npos) return dflt;
  p = txt.find(':', p); if (p == std::string::npos) return dflt;
  return strtol(txt.c_str() + p + 1, nullptr, 10);
}
}  // namespace

extern "C" int32_t demi_experiment_save(const char* dir, const demi_experiment* e) {
  if (!dir || !e || !e->externals || !e->events) return fail(nullptr, DEMI_ERR_INVALID, "demi_experiment_save: null argument");
  mkdir(dir, 0777);
  const std::string d(dir);
  bool ok = write_file(d + "/externals.bin", e->externals, (size_t)e->n_externals * sizeof(demi_ext_event)) &&
            write_file(d + "/event_trace.bin", e->events, (size_t)e->n_events * sizeof(demi_event));
  if (ok && e->dep_parent) ok = write_file(d + "/dep_parent.bin", e->dep_parent, (size_t)e->n_nodes * 2);
  if (ok && e->mcs_mask) ok = write_file(d + "/mcs.bin", e->mcs_mask, (size_t)e->mask_words * 8);
  char meta[256];
  snprintf(meta, sizeof(meta), "{\n \"format\": \"demi_b200/1\",\n \"model\": %d,\n \"model_flags\": %u,\n \"violation\": %u\n}\n",
           e->model, e->model_flags, e->violation);
  if (ok) ok = write_file(d + "/meta.json", meta, strlen(meta));
  if (!ok) return fail(nullptr, DEMI_ERR_INVALID, "demi_experiment_save: cannot write under %s", dir);
  return DEMI_OK;
}

extern "C" int32_t demi_experiment_load(const char* dir, demi_experiment* e) {
  if (!dir || !e) return fail(nullptr, DEMI_ERR_INVALID, "demi_experiment_load: null argument");
  const std::string d(dir);
  const long b_ext = file_size(d + "/externals.bin"), b_ev = file_size(d + "/event_trace.bin"),
             b_par = file_size(d + "/dep_parent.bin"), b_mcs = file_size(d + "/mcs.bin"), b_meta = file_size(d + "/meta.json");
  if (b_ext < 0 || b_ev < 0 || b_meta < 0 || b_ext % 16 || b_ev % 16)
    return fail(nullptr, DEMI_ERR_INVALID, "demi_experiment_load: %s is not an experiment directory", dir);
  e->n_externals = (uint32_t)(b_ext / 16); e->n_events = (uint32_t)(b_ev / 16);
  e->n_nodes = b_par > 0 ? (uint32_t)(b_par / 2) : 0; e->mask_words = b_mcs > 0 ? (uint32_t)(b_mcs / 8) : 0;
  std::string meta((size_t)b_meta, '\0');
  if (!read_file(d + "/meta.json", &meta[0], (size_t)b_meta)) return fail(nullptr, DEMI_ERR_INVALID, "demi_experiment_load: unreadable meta.json");
  e->model = (int32_t)json_int(meta, "model", 0); e->model_flags = (uint32_t)json_int(meta, "model_flags", 0);
  e->violation = (uint32_t)json_int(meta, "violation", 0);
  // sizes only (a first call with null / too small buffers tells the caller what to allocate)
  if (!e->externals || !e->events || e->cap_externals < e->n_externals || e->cap_events < e->n_events ||
      (e->dep_parent && e->cap_nodes < e->n_nodes) || (e->mcs_mask && e->cap_mask_words < e->mask_words))
    return fail(nullptr, DEMI_ERR_CAPACITY, "demi_experiment_load: %u externals, %u events, %u nodes, %u mask words", e->n_externals,
                e->n_events, e->n_nodes, e->mask_words);
  bool ok = read_file(d + "/externals.bin", e->externals, (size_t)b_ext) && read_file(d + "/event_trace.bin", e->events, (size_t)b_ev);
  if (ok && e->dep_parent && e->n_nodes) ok = read_file(d + "/dep_parent.bin", e->dep_parent, (size_t)e->n_nodes * 2);
  if (ok && e->mcs_mask && e->mask_words) ok = read_file(d + "/mcs.bin", e->mcs_mask, (size_t)e->mask_words * 8);
  if (!ok) return fail(nullptr, DEMI_ERR_INVALID, "demi_experiment_load: short read under %s", dir);
  return DEMI_OK;
}
