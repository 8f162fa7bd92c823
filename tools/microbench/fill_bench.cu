// fill_bench.cu - how fast can the SMs of an H100 pull L2-resident tiles into shared memory with TMA, and does
// `.multicast::cluster` lift the chip-wide cap?  (Design input for the conv kernels: their operand ring is fed by this
// path.)
//
//   mode 0: unicast, every CTA streams DISTINCT 16 KB tiles
//   mode 1: unicast, the C CTAs of a cluster request the SAME tile in the same round (does L2 merge the requests?)
//   mode 2: multicast, one CTA of the cluster requests the tile for all C CTAs (each CTA issues every C-th load)
// Every CTA receives S tiles per round (S x 16 KB ring), then the cluster synchronises and the ring is reused.
// Output: delivered GB/s = bytes landing in shared memory / time (CUDA events), per mode and cluster size.
//
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fill_bench fill_bench.cu -lcuda
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

constexpr int TILE_ROWS = 128, TILE_BYTES = TILE_ROWS * 128, STAGES = 12;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ unsigned long long gtimer() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity) {
  unsigned long long t0 = gtimer();
  while (!mbar_try_wait(bar, parity)) if (gtimer() - t0 > 1000000000ull) return false;
  return true;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_id_x() { uint32_t r; asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r)); return r; }

__global__ void __launch_bounds__(128, 1) fill_kernel(const __grid_constant__ CUtensorMap tm, int mode, int csize, int rounds,
                                                      int n_tiles, int* err, float* sink) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t bars[STAGES];
  const uint32_t base = smem_u32(smem);
  const uint32_t rank = cluster_ctarank();
  const uint32_t cid = cluster_id_x();
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) mbar_init(smem_u32(&bars[s]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  cluster_sync_all();
  uint32_t tile = (mode == 0 ? blockIdx.x : cid) * 977u;      // distinct (mode 0) or shared-by-cluster (1, 2) tile sequence
  const uint16_t mask = (uint16_t)((1u << csize) - 1u);
  for (int r = 0; r < rounds; ++r) {
    if (threadIdx.x == 0) {
      for (int s = 0; s < STAGES; ++s) {
        const uint32_t bar = smem_u32(&bars[s]);
        mbar_expect_tx(bar, TILE_BYTES);
        const int row = (int)((tile + (uint32_t)s * 131u) % (uint32_t)n_tiles) * TILE_ROWS;
        const uint32_t dst = base + s * TILE_BYTES;
        if (mode == 2) {
          if ((uint32_t)(s % csize) == rank)
            asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
                         ::"r"(dst), "l"(reinterpret_cast<uint64_t>(&tm)), "r"(bar), "r"(0), "r"(row), "h"(mask) : "memory");
        } else {
          asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                       ::"r"(dst), "l"(reinterpret_cast<uint64_t>(&tm)), "r"(bar), "r"(0), "r"(row) : "memory");
        }
      }
      for (int s = 0; s < STAGES; ++s)
        if (!mbar_wait(smem_u32(&bars[s]), (uint32_t)(r & 1))) { atomicExch(err, 1 + s); break; }
    }
    tile += 7919u;
    __syncthreads();
    if (csize > 1) cluster_sync_all();     // nobody refills a peer's ring before the peer has seen this round land
  }
  if (sink && threadIdx.x == 0) sink[blockIdx.x] = (float)smem[blockIdx.x & 1023];
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// Experiment 2: G CTAs share one tile sequence (what the N-tile / weight operand of a conv does: many CTAs stream the SAME
// tiles); rot = 1 makes the sharers walk the round's tiles in rotated order so they never ask for the same tile at the
// same moment.  No clusters, no multicast.
__global__ void __launch_bounds__(128, 1) share_kernel(const __grid_constant__ CUtensorMap tm, int group, int rot, int rounds,
                                                       int n_tiles, int* err, float* sink) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t bars[STAGES];
  const uint32_t base = smem_u32(smem);
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) mbar_init(smem_u32(&bars[s]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint32_t gid = blockIdx.x / group, member = blockIdx.x % group;
  uint32_t tile = gid * 977u;
  for (int r = 0; r < rounds; ++r) {
    if (threadIdx.x == 0) {
      for (int s = 0; s < STAGES; ++s) {
        const uint32_t bar = smem_u32(&bars[s]);
        mbar_expect_tx(bar, TILE_BYTES);
        const uint32_t which = rot ? (uint32_t)(s + member) % STAGES : (uint32_t)s;
        const int row = (int)((tile + which * 131u) % (uint32_t)n_tiles) * TILE_ROWS;
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                     ::"r"(base + s * TILE_BYTES), "l"(reinterpret_cast<uint64_t>(&tm)), "r"(bar), "r"(0), "r"(row) : "memory");
      }
      for (int s = 0; s < STAGES; ++s)
        if (!mbar_wait(smem_u32(&bars[s]), (uint32_t)(r & 1))) { atomicExch(err, 1 + s); break; }
    }
    tile += 7919u;
    __syncthreads();
  }
  if (sink && threadIdx.x == 0) sink[blockIdx.x] = (float)smem[blockIdx.x & 1023];
}

int main(int argc, char** argv) {
  const size_t total_mb = argc > 1 ? atoi(argv[1]) : 64;     // working set (L2-resident by default)
  const int rounds = argc > 2 ? atoi(argv[2]) : 200;
  int dev = 0, sms = 0;
  CK(cudaSetDevice(dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int n_tiles = (int)(total_mb * 1024 * 1024 / TILE_BYTES);
  void* buf = nullptr;
  CK(cudaMalloc(&buf, (size_t)n_tiles * TILE_BYTES));
  CK(cudaMemset(buf, 1, (size_t)n_tiles * TILE_BYTES));
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  CUtensorMap tm;
  cuuint64_t dims[2] = {64, (cuuint64_t)n_tiles * TILE_ROWS};
  cuuint64_t strides[1] = {128};
  cuuint32_t box[2] = {64, TILE_ROWS}, es[2] = {1, 1};
  CUresult cr = ((PFN_encodeTiled)fn)(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, buf, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) { printf("encode failed %d\n", (int)cr); return 1; }
  int* err = nullptr;
  float* sink = nullptr;
  CK(cudaMalloc(&err, 4));
  CK(cudaMalloc(&sink, 4096 * 4));
  const size_t smem = (size_t)STAGES * TILE_BYTES + 1024;
  CK(cudaFuncSetAttribute(fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CK(cudaFuncSetAttribute(fill_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  printf("# TMA fill benchmark: %d SMs, working set %zu MB, %d rounds x %d tiles x 16 KB per CTA\n", sms, total_mb, rounds, STAGES);
  printf("# mode csize grid  time_ms  delivered_GBs  per_SM_GBs\n");
  const int modes[] = {0, 1, 2};
  const int csizes[] = {1, 2, 4, 8};
  for (int grid_div = 1; grid_div <= 4; grid_div *= 4) {     // all SMs, then a quarter of them (per-SM cap)
    for (int mi = 0; mi < 3; ++mi) {
      for (int ci = 0; ci < 4; ++ci) {
        const int mode = modes[mi], cs = csizes[ci];
        if (mode == 0 && cs != 1) continue;
        if (mode != 0 && cs == 1) continue;
        int grid = (sms / grid_div) / cs * cs;
        if (grid < cs) continue;
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof cfg);
        cfg.gridDim = dim3(grid, 1, 1);
        cfg.blockDim = dim3(128, 1, 1);
        cfg.dynamicSmemBytes = smem;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        CK(cudaMemset(err, 0, 4));
        float best = 1e30f;
        for (int rep = 0; rep < 4; ++rep) {
          CK(cudaEventRecord(e0));
          cudaError_t le = cudaLaunchKernelEx(&cfg, fill_kernel, tm, mode, cs, rounds, n_tiles, err, sink);
          if (le != cudaSuccess) { printf("launch failed (mode %d csize %d grid %d): %s\n", mode, cs, grid, cudaGetErrorString(le)); cudaGetLastError(); best = -1; break; }
          CK(cudaEventRecord(e1));
          CK(cudaEventSynchronize(e1));
          float ms = 0;
          CK(cudaEventElapsedTime(&ms, e0, e1));
          if (rep > 0 && ms < best) best = ms;
        }
        int herr = 0;
        CK(cudaMemcpy(&herr, err, 4, cudaMemcpyDeviceToHost));
        if (best < 0) continue;
        const double bytes = (double)grid * rounds * STAGES * TILE_BYTES;
        printf("  %d    %d     %3d  %8.3f  %10.1f  %8.1f %s\n", mode, cs, grid, best, bytes / best / 1e6, bytes / best / 1e6 / grid,
               herr ? "TIMEOUT" : "");
      }
    }
  }
  CK(cudaFuncSetAttribute(share_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  printf("# experiment 2: sharing groups (no clusters). group rot grid time_ms delivered_GBs per_SM_GBs\n");
  const int groups[] = {1, 2, 4, 8, 16, sms / 4, sms};   // up to every SM reading the same tiles
  for (int gi = 0; gi < 7; ++gi) {
    for (int rot = 0; rot < 2; ++rot) {
      const int g = groups[gi];
      if (g == 1 && rot) continue;
      const int grid = sms / g * g;
      CK(cudaMemset(err, 0, 4));
      float best = 1e30f;
      for (int rep = 0; rep < 4; ++rep) {
        CK(cudaEventRecord(e0));
        share_kernel<<<grid, 128, smem>>>(tm, g, rot, rounds, n_tiles, err, sink);
        CK(cudaGetLastError());
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        if (rep > 0 && ms < best) best = ms;
      }
      int herr = 0;
      CK(cudaMemcpy(&herr, err, 4, cudaMemcpyDeviceToHost));
      const double bytes = (double)grid * rounds * STAGES * TILE_BYTES;
      printf("  %3d   %d   %3d  %8.3f  %10.1f  %8.1f %s\n", g, rot, grid, best, bytes / best / 1e6, bytes / best / 1e6 / grid, herr ? "TIMEOUT" : "");
    }
  }
  return 0;
}
