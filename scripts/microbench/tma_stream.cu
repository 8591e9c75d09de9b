// Microbenchmark (diagnostic, not product): what read bandwidth can per-warp cp.async.bulk rings reach on this GPU, as a
// function of stage size, ring depth and resident warps?  The dense PCG operator (k_matvec_small_tma) streams its panels
// with exactly this structure (DESIGN.md section 11.1); this sweep separates "structure of the stream" from "everything
// else".
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tma_stream tma_stream.cu && ./tma_stream [GiB]
//
// Prints one line per configuration: GB/s read.  Baselines: grid-stride 16-byte loads, cudaMemcpy device-to-device.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { std::printf("%s: %s\n", #x, cudaGetErrorString(e)); std::exit(1); } } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy, bool hint) {
  if (hint)
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
                 : "memory");
  else
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(smem_u32(b)), "r"(parity) : "memory");
  } while (!ok);
}

// Every warp owns a private ring of NS stages; chunk q of CHUNK bytes (a "matvec item") is read by warp q mod nwarps in
// stages of STAGE bytes -- the access pattern of k_matvec_small_tma.  `sink` keeps one word per stage alive.
template <int WARPS, int NS, int STAGE>
__global__ void __launch_bounds__(WARPS * 32) k_ring(const unsigned char* __restrict__ src, size_t chunk_bytes, long long nchunks, int hint, float* sink) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t bars_all[WARPS][NS];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* ring = smem + (size_t)wib * NS * STAGE;
  uint64_t* bars = bars_all[wib];
  if (lane == 0) {
    for (int s = 0; s < NS; ++s) mbar_init(&bars[s], 1);
    mbar_fence_init();
  }
  __syncwarp();
  uint64_t policy;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
  const long long stride = (long long)gridDim.x * WARPS;
  const long long first = (long long)blockIdx.x * WARPS + wib;
  const int stages_per_chunk = (int)(chunk_bytes / STAGE);
  // producer cursor
  long long pq = first; int ps = 0; unsigned issued = 0, consumed = 0;
  auto produce = [&]() -> bool {
    if (pq >= nchunks) return false;
    if (lane == 0) {
      const unsigned slot = issued % NS;
      mbar_expect_tx(&bars[slot], STAGE);
      bulk_g2s(ring + (size_t)slot * STAGE, src + (size_t)pq * chunk_bytes + (size_t)ps * STAGE, STAGE, &bars[slot], policy, hint != 0);
    }
    ++issued;
    if (++ps == stages_per_chunk) { ps = 0; pq += stride; }
    return true;
  };
  for (int s = 0; s < NS; ++s) if (!produce()) break;
  float acc = 0;
  while (consumed < issued) {
    const unsigned slot = consumed % NS;
    mbar_wait(&bars[slot], (consumed / NS) & 1u);
    acc += reinterpret_cast<const float*>(ring + (size_t)slot * STAGE)[lane];
    ++consumed;
    __syncwarp();
    produce();
  }
  if (acc == 123.456f) sink[0] = acc;
}

__global__ void k_ldg(const float4* __restrict__ src, size_t n4, float* sink) {
  float acc = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(src + i);
    acc += v.x + v.y + v.z + v.w;
  }
  if (acc == 123.456f) sink[0] = acc;
}

static float time_ms(cudaEvent_t a, cudaEvent_t b) { float ms = 0; CK(cudaEventElapsedTime(&ms, a, b)); return ms; }

template <int WARPS, int NS, int STAGE>
void run_ring(const unsigned char* d, size_t bytes, size_t chunk, int hint, int sms, float* sink) {
  const size_t smem = (size_t)WARPS * NS * STAGE;
  if (smem > 220 * 1024) return;
  CK(cudaFuncSetAttribute((k_ring<WARPS, NS, STAGE>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int bps = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, (k_ring<WARPS, NS, STAGE>), WARPS * 32, smem));
  if (bps < 1) return;
  const long long nchunks = (long long)(bytes / chunk);
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  for (int cap : {0, 5, 3, 2, 1}) {  // 0 = as many blocks per SM as fit
    const int use = cap == 0 ? bps : cap;
    if (use > bps || (cap != 0 && cap == bps)) continue;
    const int grid = sms * use;
    k_ring<WARPS, NS, STAGE><<<grid, WARPS * 32, smem>>>(d, chunk, nchunks, hint, sink);
    CK(cudaEventRecord(a));
    const int reps = 5;
    for (int r = 0; r < reps; ++r) k_ring<WARPS, NS, STAGE><<<grid, WARPS * 32, smem>>>(d, chunk, nchunks, hint, sink);
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    const double gbs = (double)nchunks * chunk * reps / (time_ms(a, b) * 1e-3) / 1e9;
    std::printf("ring  stage %6d B  x%d stages  %2d warps/SM (%d blocks x %d)  chunk %7zu B  hint %d : %8.1f GB/s\n", STAGE, NS, use * WARPS, use, WARPS,
                chunk, hint, gbs);
  }
  CK(cudaEventDestroy(a)); CK(cudaEventDestroy(b));
}

int main(int argc, char** argv) {
  const double gib = argc > 1 ? std::atof(argv[1]) : 2.0;
  const size_t bytes = (size_t)(gib * (1ull << 30)) / (1 << 20) * (1 << 20);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  std::printf("%s, %d SMs, buffer %.2f GiB (L2 %d MB)\n", prop.name, sms, bytes / double(1ull << 30), prop.l2CacheSize >> 20);
  unsigned char *d = nullptr, *d2 = nullptr;
  float* sink = nullptr;
  CK(cudaMalloc(&d, bytes)); CK(cudaMalloc(&d2, bytes)); CK(cudaMalloc(&sink, 4));
  CK(cudaMemset(d, 1, bytes)); CK(cudaMemset(d2, 0, bytes));
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  {
    CK(cudaMemcpy(d2, d, bytes, cudaMemcpyDeviceToDevice));
    CK(cudaEventRecord(a));
    for (int r = 0; r < 5; ++r) CK(cudaMemcpyAsync(d2, d, bytes, cudaMemcpyDeviceToDevice));
    CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
    std::printf("cudaMemcpy D2D: %8.1f GB/s copied (read + write = 2x)\n", (double)bytes * 5 / (time_ms(a, b) * 1e-3) / 1e9);
  }
  for (int bpsm : {8, 16, 32}) {
    k_ldg<<<sms * bpsm, 256>>>((const float4*)d, bytes / 16, sink);
    CK(cudaEventRecord(a));
    for (int r = 0; r < 5; ++r) k_ldg<<<sms * bpsm, 256>>>((const float4*)d, bytes / 16, sink);
    CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
    std::printf("ldg.128 grid-stride, %2d blocks/SM x 256 threads: %8.1f GB/s\n", bpsm, (double)bytes * 5 / (time_ms(a, b) * 1e-3) / 1e9);
  }
  // the operator's configuration first (4 warps, 2 x 4608 B), then the sweep; chunk = bytes one warp streams contiguously
  for (int hint : {1, 0}) {
    for (size_t chunk : {(size_t)18432, (size_t)73728}) {
      run_ring<4, 2, 4608>(d, bytes, chunk, hint, sms, sink);
      run_ring<4, 3, 4608>(d, bytes, chunk, hint, sms, sink);
      run_ring<4, 4, 4608>(d, bytes, chunk, hint, sms, sink);
      run_ring<4, 2, 9216>(d, bytes, chunk, hint, sms, sink);
      run_ring<4, 3, 9216>(d, bytes, chunk, hint, sms, sink);
      run_ring<4, 2, 18432>(d, bytes, chunk, hint, sms, sink);
      run_ring<2, 2, 18432>(d, bytes, chunk, hint, sms, sink);
      run_ring<4, 4, 2304>(d, bytes, chunk, hint, sms, sink);
      run_ring<8, 2, 4608>(d, bytes, chunk, hint, sms, sink);
    }
  }
  CK(cudaGetLastError());
  std::printf("done\n");
  return 0;
}
