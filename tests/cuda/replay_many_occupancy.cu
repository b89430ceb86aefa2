// Resident blocks per SM of the multi-trace K2 kernel next to the single-trace one, per model, at the block size and
// dynamic shared memory the C ABI launches them with (replay_block, capi_replay.cu).  Prints one line per model:
// "<model> <single> <many>".
#include <cstdio>
#include "../../demi_b200/csrc/replay_kernel.cuh"
#include "../../demi_b200/csrc/models/model_ir.cuh"

using namespace demi;

template <class MODEL>
static int report(const char* name) {
  constexpr int BD = replay_block<MODEL>;
  const size_t smem = (size_t)ReplayMachine<MODEL, BD>::WORDS * BD * sizeof(uint32_t);
  const void* fns[2] = {(const void*)replay_lane_kernel<MODEL, BD, false, false>, (const void*)replay_many_kernel<MODEL, BD>};
  int bps[2] = {0, 0};
  for (int k = 0; k < 2; k++) {
    if (cudaFuncSetAttribute(fns[k], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps[k], fns[k], BD, smem) != cudaSuccess) return 1;
  }
  printf("%s %d %d\n", name, bps[0], bps[1]);
  return 0;
}

int main() {
  int rc = report<PingPong3>("pingpong3") | report<Raft5>("raft5") | report<Bcast32>("bcast32") | report<IrModel>("ir");
  return rc;
}
