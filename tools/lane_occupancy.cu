// Resident CTAs per SM of the Telegram lane emitter (tg_emit_lane_kernel) as the CUDA runtime computes them for the
// build's LB_LANE / LANE_STAGE, with the registers, local memory and dynamic shared memory behind that number.
// Built by tools/variants.sh next to each library variant; run on the GPU box:  build_variants/lane_occupancy_<variant>
#include "../distributed_crawler_b200/csrc/tgingest.cu"

#include <cstdio>

int main() {
  using namespace tgi;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, 0) != cudaSuccess) {
    fprintf(stderr, "no CUDA device\n");
    return 1;
  }
  cudaFuncAttributes fa;
  int ctas = 0;
  const int smem = (int)sizeof(LaneShared);
  if (cudaFuncSetAttribute(tg_emit_lane_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess ||
      cudaFuncGetAttributes(&fa, tg_emit_lane_kernel) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, tg_emit_lane_kernel, CTA_THREADS, smem) != cudaSuccess) {
    fprintf(stderr, "occupancy query failed\n");
    return 1;
  }
  printf("{\"device\": \"%s\", \"LB_LANE\": %d, \"LANE_STAGE\": %d, \"registers\": %d, \"local_bytes\": %zu, "
         "\"lane_shared_bytes\": %d, \"reserved_smem_per_cta\": %zu, \"smem_per_sm\": %zu, \"ctas_per_sm\": %d}\n",
         prop.name, LB_LANE, LANE_STAGE, fa.numRegs, fa.localSizeBytes, smem, prop.reservedSharedMemPerBlock,
         prop.sharedMemPerMultiprocessor, ctas);
  return 0;
}
