// Micro-benchmark: the weight requests of the chained kernels (chain.cuh) at the shapes they use, on CTAs that each stream
// the same L2-resident 256 x 256 fp32 matrix (256 KB) through `stages` shared-memory slots (stages - 1 requests in flight,
// like the chain pipeline with one slot being read).  Compares
//   2d32   2-D tensor map, box {32 k, 256 n}, SWIZZLE_128B            -- one 32 KB forward chunk (the control)
//   3d64   3-D tensor map, dims (32 k, 256 n, 8 k-chunks), strides (pitch, 128 B), box {32, 256, 2}, SWIZZLE_128B
//          -- two consecutive forward chunks in one 64 KB request
//   1d32   cp.async.bulk of 32 rows (32 KB)                             -- one backward chunk
//   1d64   cp.async.bulk of 64 rows (64 KB)                             -- two backward chunks in one request
// and reports cycles per 32 KB.  Is the chunk cadence bound by the number of requests per SM or by their bytes?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_pair_rate tma_pair_rate.cu && ./tma_pair_rate
#include <cstdio>
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while (0)

constexpr int THREADS = 256, N = 256, KDIM = 256;
enum { M_2D32 = 0, M_3D64 = 1, M_1D32 = 2, M_1D64 = 3 };
static const char* kName[] = {"2d32", "3d64", "1d32", "1d64"};
static const int kBytes[] = {32768, 65536, 32768, 65536};

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(b), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_expect(uint32_t b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory"); }
__device__ __forceinline__ bool mbar_try(uint32_t b, uint32_t ph) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(b), "r"(ph) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t b, uint32_t ph) {
  const long long t0 = clock64();
  while (!mbar_try(b, ph)) if (clock64() - t0 > 2000000000LL) __trap();
}

__global__ void __launch_bounds__(THREADS, 1) stream_kernel(const __grid_constant__ CUtensorMap tm2, const __grid_constant__ CUtensorMap tm3,
                                                            const float* __restrict__ W, int mode, int nstage, int total,
                                                            long long* out_cycles, float* sink) {
  extern __shared__ __align__(1024) uint8_t sm_raw[];
  uint8_t* sm = sm_raw + ((1024u - (s32(sm_raw) & 1023u)) & 1023u);
  const int bytes = (mode == M_3D64 || mode == M_1D64) ? 65536 : 32768;
  const int per_pass = (KDIM * N * 4) / bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(sm + (size_t)nstage * bytes);
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int i = 0; i < nstage; ++i) mbar_init(s32(full + i), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  int issued = 0;
  auto issue = [&]() {
    if (tid == 0 && issued < total) {
      const int slot = issued % nstage, p = issued % per_pass;
      const uint32_t bar = s32(full + slot), dst = s32(sm + (size_t)slot * bytes);
      mbar_expect(bar, bytes);
      if (mode == M_2D32) {
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                     ::"r"(dst), "l"(&tm2), "r"(bar), "r"(32 * p), "r"(0) : "memory");
      } else if (mode == M_3D64) {
        asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                     ::"r"(dst), "l"(&tm3), "r"(bar), "r"(0), "r"(0), "r"(2 * p) : "memory");
      } else {
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(dst), "l"(reinterpret_cast<const char*>(W) + (size_t)p * bytes), "r"(bytes), "r"(bar) : "memory");
      }
      ++issued;
    }
  };
  for (int i = 0; i < nstage - 1; ++i) issue();
  float acc = 0.f;
  const long long t0 = clock64();
  for (int g = 0; g < total; ++g) {
    const int slot = g % nstage;
    mbar_wait(s32(full + slot), (uint32_t)((g / nstage) & 1));
    __syncthreads();
    if (tid == 0) issue();
    const float4 v = *reinterpret_cast<const float4*>(sm + (size_t)slot * bytes + tid * 16);
    acc += v.x + v.y + v.z + v.w;
  }
  const long long t1 = clock64();
  if (tid == 0 && blockIdx.x == 0) *out_cycles = t1 - t0;
  if (acc == 12345.678f) *sink = acc;
}

// Each 3-D request must land as two consecutive swizzled [256 n][32 k] chunks, i.e. exactly what two 2-D requests deliver.
__global__ void compare_kernel(const __grid_constant__ CUtensorMap tm2, const __grid_constant__ CUtensorMap tm3, int* mismatches) {
  extern __shared__ __align__(1024) uint8_t sm_raw[];
  uint8_t* sm = sm_raw + ((1024u - (s32(sm_raw) & 1023u)) & 1023u);
  uint64_t* bar = reinterpret_cast<uint64_t*>(sm + 2 * 65536);
  const uint32_t b = s32(bar);
  if (threadIdx.x == 0) { mbar_init(b, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  for (int p = 0; p < KDIM / 64; ++p) {
    if (threadIdx.x == 0) {
      mbar_expect(b, 2 * 65536);
      for (int h = 0; h < 2; ++h)
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                     ::"r"(s32(sm + h * 32768)), "l"(&tm2), "r"(b), "r"(64 * p + 32 * h), "r"(0) : "memory");
      asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                   ::"r"(s32(sm + 65536)), "l"(&tm3), "r"(b), "r"(0), "r"(0), "r"(2 * p) : "memory");
    }
    mbar_wait(b, (uint32_t)(p & 1));
    int bad = 0;
    for (int i = threadIdx.x; i < 16384; i += blockDim.x)
      bad += reinterpret_cast<const uint32_t*>(sm)[i] != reinterpret_cast<const uint32_t*>(sm + 65536)[i];
    if (bad) atomicAdd(mismatches, bad);
    __syncthreads();
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main() {
  void* fp = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
    printf("cuTensorMapEncodeTiled not available\n");
    return 1;
  }
  EncodeTiledFn enc = (EncodeTiledFn)fp;
  float* W; long long* d_cyc; float* d_sink; int* d_bad;
  CK(cudaMalloc(&W, KDIM * N * 4));
  CK(cudaMalloc(&d_cyc, 8)); CK(cudaMalloc(&d_sink, 4)); CK(cudaMalloc(&d_bad, 4));
  {
    float h[KDIM * N];
    for (int i = 0; i < KDIM * N; ++i) h[i] = (float)i;
    CK(cudaMemcpy(W, h, sizeof(h), cudaMemcpyHostToDevice));
  }
  CUtensorMap tm2, tm3;
  const cuuint32_t estr[3] = {1u, 1u, 1u};
  {  // W [256 n][256 k], box {32 k, 256 n}
    const cuuint64_t dims[2] = {KDIM, N}, strides[1] = {KDIM * 4};
    const cuuint32_t box[2] = {32, N};
    CUresult r = enc(&tm2, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, W, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { printf("2-D map: error %d\n", (int)r); return 1; }
  }
  {  // the same matrix as (k within chunk, n, k-chunk)
    const cuuint64_t dims[3] = {32, N, KDIM / 32}, strides[2] = {KDIM * 4, 128};
    const cuuint32_t box[3] = {32, N, 2};
    CUresult r = enc(&tm3, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, W, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { printf("3-D map: error %d\n", (int)r); return 1; }
  }
  CK(cudaFuncSetAttribute(compare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 65536 + 1024 + 64));
  CK(cudaMemset(d_bad, 0, 4));
  compare_kernel<<<1, THREADS, 2 * 65536 + 1024 + 64>>>(tm2, tm3, d_bad);
  CK(cudaDeviceSynchronize());
  int bad = -1;
  CK(cudaMemcpy(&bad, d_bad, 4, cudaMemcpyDeviceToHost));
  printf("3-D 64 KB request vs two 2-D 32 KB requests: %d mismatching words\n", bad);

  const int smem_max = 3 * 65536 + 1024 + 64;
  CK(cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
  for (int ctas : {8, 128}) {
    printf("%d CTAs:\n", ctas);
    for (int mode : {M_2D32, M_3D64, M_1D32, M_1D64})
      for (int nstage : {2, 3}) {
        const int total = 32 * (KDIM * N * 4 / kBytes[mode]);
        const int smem = nstage * kBytes[mode] + 1024 + 64;
        for (int it = 0; it < 3; ++it) stream_kernel<<<ctas, THREADS, smem>>>(tm2, tm3, W, mode, nstage, total, d_cyc, d_sink);
        CK(cudaDeviceSynchronize());
        long long cyc = 0;
        CK(cudaMemcpy(&cyc, d_cyc, 8, cudaMemcpyDeviceToHost));
        const double per_req = (double)cyc / total, per32 = per_req * 32768.0 / kBytes[mode];
        printf("  %s, %d stages: %7.1f cycles per request, %7.1f per 32 KB  (%5.1f B/clk/SM)\n", kName[mode], nstage, per_req, per32,
               32768.0 / per32);
      }
  }
  return 0;
}
