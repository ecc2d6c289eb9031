// wgmma (Hopper warpgroup tensor core) grouped GEMM for the hidden layers of the SAC step, at fp32-class accuracy via the
// 3xTF32 split:  x = hi + lo (hi = top 19 bits of x, lo = x - hi, exact in fp32),  D += A_hi*B_hi + A_hi*B_lo + A_lo*B_hi.
//
// One CTA = one 128 x BN output tile (BN = 64 / 128 / 160) of one problem (blockIdx.z = problem x replica), two
// warpgroups (rows 0-63 / 64-127 of the tile); 256 threads leave each thread up to 255 registers for its accumulators.
//   TMA         thread 0 issues one cp.async.bulk.tensor 2-D box per operand and 32-wide k chunk, straight from the row-major
//               activation / weight / gradient buffers into a stage's raw area, as soon as both warpgroups' MMAs have
//               released that stage; out-of-range rows and columns are zero-filled by the TMA unit (ragged 400-wide
//               layers, tails).  K-major operands arrive SWIZZLE_128B (already the wgmma K-major layout), MN-major ones
//               unswizzled [32 k][rows].
//   split       both warpgroups split every landed chunk together: hi and
//               lo are written in the K-major SWIZZLE_128B layout wgmma reads (wgmma takes tf32 operands only K-major, so
//               the MN-major DGRAD / WGRAD operands are transposed here on the way).  Each warpgroup then issues
//               12 wgmma.m64nBNk8 per chunk into a register accumulator and, while those run, splits the next chunk.
//               The PAIRED 128-wide tile issues 8 instead: the lo tile of B lies right behind its hi tile, so one
//               m64n256k8 computes A_hi * [B_hi ; B_lo] into [main | cross] and one m64n128k8 adds A_lo * B_hi into
//               cross.  It reads A_hi once per k step instead of twice, but the two shapes write overlapping accumulator
//               registers, so each MMA completes before the next is issued (PTX orders accumulator accesses only between
//               wgmma of one shape), and its 256-column accumulator next to the running total leaves ptxas too few
//               registers to pipeline them anyway; it measured slower on an H100 (3.1k against 2.65k cycles per chunk),
//               so it runs only when B200SAC_TC_PAIR128=1 selects it.
//   accumulate  each chunk's products are summed by the tensor core into a fresh accumulator and added to the running
//               total with an ordinary round-to-nearest fp32 add (the tensor core's own accumulation is not IEEE
//               round-to-nearest, so its error is kept to one 32-deep chunk).  Keeps the result within ~1e-6 of fp64.
//   epilogue    registers -> bias+ReLU | ReLU' mask | plain -> global; the weight-gradient kind also emits the bias
//               gradient (column sums of dY), summed by the splitting threads in a fixed order.
// The three GEMM kinds only differ in operand majors, exactly as in gemm_simt.cuh:
//   FWD   A = X  [M][K] K-major,  B = W [N][K] K-major
//   DGRAD A = dY [M][K] K-major,  B = W [K][N] MN-major
//   WGRAD A = dY [K][M] MN-major, B = X [K][N] MN-major
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "gemm_simt.cuh"

namespace bsac {

constexpr int TC_BM = 128, TC_BK = 32;
constexpr int TC_A_BYTES = TC_BM * TC_BK * 4;                  // 16 KiB
constexpr int TC_THREADS = 256;                                // two warpgroups
constexpr int TC_BSUM_BYTES = 8 * TC_BM * 4;                   // [8 partials][128 m] fp32

// Tile widths: 128x64 (many CTAs: latency-critical small problems), 128x128 (the 400-wide shapes: each wgmma reads its
// A operand once for twice the columns; paired or not) and 128x160 (400 = 3 x 160 - 80: launch groups whose 128-wide tiling needs a
// second wave of CTAs but whose 160-wide tiling fits one).  A stage holds raw, hi and lo copies of both operand tiles.
template <int BN>
struct TcCfg {
  static constexpr int kBN = BN;
  static constexpr int kBBytes = BN * TC_BK * 4;                           // 8 / 16 / 20 KiB
  static constexpr int kStageBytes = 3 * (TC_A_BYTES + kBBytes);           // 72 / 96 / 108 KiB
  static constexpr int kStages = BN == 64 ? 3 : 2;
  static constexpr int kSmemBytes = kStages * kStageBytes + TC_BSUM_BYTES + 256 + 1024;   // + barriers + align slack
  static_assert(kSmemBytes <= 232448, "shared memory");
  static_assert(BN % 32 == 0 && kBBytes % 1024 == 0, "tile width");
};

struct alignas(128) TcProb {
  CUtensorMap tmA;
  CUtensorMap tmB;
  const float* bias;
  const float* mask;
  float* C;
  float* C2;
  int M, N, K;
  int ldc, ldmask;
  int mode, relu;
  int a_mn, b_mn;
  long long* dbg;      // optional clock64() timeline of CTA (0,0) (b200sac_tc_gemm_timeline)
};

#define TC_STAMP(i) do { if (dbg) dbg[(i)] = clock64(); } while (0)

// ---- PTX wrappers ---------------------------------------------------------------------------
B200_D uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

B200_D void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
B200_D void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
B200_D void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
B200_D bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must become a trapped launch, never a hung GPU.
B200_D void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
B200_D void tma_load_2d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}

B200_D void stg_f32(float* p, float v) { asm volatile("st.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory"); }
B200_D float ldg_f32(const float* p) {
  float v;
  asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}

// wgmma shared-memory matrix descriptor for a K-major SWIZZLE_128B tile: rows of 128 B (32 tf32), 8-row groups 1024 B
// apart (stride byte offset), leading byte offset unused; layout type 1 = 128-B swizzle.  The tile must be 1024-B aligned;
// the k step of 8 tf32 advances the start address by 32 B inside the swizzle atom.
B200_D uint64_t wg_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
B200_D void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
B200_D void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
B200_D void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 operands from shared memory, fp32 accumulator in registers:
// thread t of the warpgroup holds rows 16 (t/32) + (t%32)/4 (+8) and columns 8 j + 2 (t%4) (+1) in d[4 j .. 4 j + 3].
template <int N> struct Wgmma;
template <> struct Wgmma<64> {
  static B200_D void mma(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d));
  }
};
template <> struct Wgmma<128> {
  static B200_D void mma(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(scale_d));
  }
};
template <> struct Wgmma<160> {
  static B200_D void mma(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %82, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n160k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, %80, %81, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
        : "l"(a), "l"(b), "r"(scale_d));
  }
};

template <> struct Wgmma<256> {
  static B200_D void mma(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a), "l"(b), "r"(scale_d));
  }
};

template <int N>
B200_D void wg_fence_acc(float* d) {
#pragma unroll
  for (int i = 0; i < N / 2; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Split one landed operand tile of ROWS rows x 32 k into hi / lo, both K-major SWIZZLE_128B (16-B chunk c of row r at
// r * 128 + ((c ^ (r & 7)) << 4)).  A K-major raw tile has that layout already; an MN-major raw tile is [32 k][ROWS].
template <int ROWS>
B200_D void tc_split(const uint8_t* raw, uint8_t* hi, uint8_t* lo, bool mn, int t) {
  constexpr int U = ROWS * 8 / TC_THREADS;                  // 16-B units per thread
  auto trunc19 = [](float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); };
  float4 v[U];
  int off[U];
  if (!mn) {
#pragma unroll
    for (int i = 0; i < U; ++i) {
      off[i] = (t + TC_THREADS * i) * 16;
      v[i] = *reinterpret_cast<const float4*>(raw + off[i]);
    }
  } else {                                                     // a warp takes 32 consecutive rows of one 4-k column
    const float* rf = reinterpret_cast<const float*>(raw);
#pragma unroll
    for (int i = 0; i < U; ++i) {
      const int u = t + TC_THREADS * i, r = u % ROWS, c = u / ROWS;
      v[i] = make_float4(rf[(4 * c) * ROWS + r], rf[(4 * c + 1) * ROWS + r], rf[(4 * c + 2) * ROWS + r], rf[(4 * c + 3) * ROWS + r]);
      off[i] = r * 128 + ((c ^ (r & 7)) << 4);
    }
  }
#pragma unroll
  for (int i = 0; i < U; ++i) {
    const float4 h = make_float4(trunc19(v[i].x), trunc19(v[i].y), trunc19(v[i].z), trunc19(v[i].w));
    *reinterpret_cast<float4*>(hi + off[i]) = h;
    *reinterpret_cast<float4*>(lo + off[i]) = make_float4(v[i].x - h.x, v[i].y - h.y, v[i].z - h.z, v[i].w - h.w);
  }
}

template <int BN, bool PAIRED>
// sched: an actor-side launch's replica-0 schedule word (replica blockIdx.z / G at sched_stride ints further; the launch is
// skipped on critic-only steps); null = always runs.
__global__ void __launch_bounds__(TC_THREADS, 1) gemm_tc_kernel(const TcProb* __restrict__ probs, const int* sched_base, int G,
                                                                int sched_stride) {
  static_assert(!PAIRED || BN == 128, "the paired variant is the 128-wide tile");
  constexpr int NACC = PAIRED ? 2 * BN : BN;                   // accumulator columns: [main | cross] when paired
  using Cfg = TcCfg<BN>;
  constexpr int B_BYTES = Cfg::kBBytes, STAGE = Cfg::kStageBytes, S = Cfg::kStages;
  constexpr int HI_A = TC_A_BYTES, LO_A = 2 * TC_A_BYTES, RAW_B = 3 * TC_A_BYTES, HI_B = RAW_B + B_BYTES, LO_B = RAW_B + 2 * B_BYTES;
  const int sched = sched_base ? sched_word(sched_base + (int)(blockIdx.z / G) * sched_stride) : SCHED_ACTOR;   // (sched_word)
  KStamp ks_;
  const TcProb* P = probs + blockIdx.z;
  extern __shared__ uint8_t smem_raw[];
  const int M = P->M, N = P->N, K = P->K;
  const int m0 = blockIdx.y * TC_BM, n0 = blockIdx.x * BN;
  if (m0 >= M || n0 >= N) return;

  const uint32_t raw_s = smem_u32(smem_raw);
  const uint32_t base = (raw_s + 1023u) & ~1023u;             // SWIZZLE_128B tiles need 1024-B alignment
  uint8_t* gbase = smem_raw + (base - raw_s);
  float* bsum_g = reinterpret_cast<float*>(gbase + S * STAGE);
  const uint32_t bars = base + S * STAGE + TC_BSUM_BYTES;
  auto full_bar = [&](int s) { return bars + 8u * s; };       // TMA landed
  auto empty_bar = [&](int s) { return bars + 8u * (S + s); };  // both warpgroups' MMAs on the stage completed

  const int lane = threadIdx.x % 32;
  const int nk = (K + TC_BK - 1) / TC_BK;
  long long* dbg = (blockIdx.x == 0 && blockIdx.y == 0 && lane == 0) ? P->dbg : nullptr;
  if (threadIdx.x == 0) TC_STAMP(0);
  const int a_mn = P->a_mn, b_mn = P->b_mn;

  const int t = threadIdx.x, wg = t / 128;
  auto load = [&](int kc) {                                    // thread 0: TMA of chunk kc into stage kc % S
    const int s = kc % S;
    mbar_expect_tx(full_bar(s), TC_A_BYTES + B_BYTES);
    const uint32_t st = base + (uint32_t)s * STAGE;
    const int k0 = kc * TC_BK;
    if (!a_mn) tma_load_2d(st, &P->tmA, k0, m0, full_bar(s));
    else tma_load_2d(st, &P->tmA, m0, k0, full_bar(s));
    if (!b_mn) tma_load_2d(st + RAW_B, &P->tmB, k0, n0, full_bar(s));
    else tma_load_2d(st + RAW_B, &P->tmB, n0, k0, full_bar(s));
    if (kc < 16) TC_STAMP(2 + kc);
  };
  if (t == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&P->tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&P->tmB) : "memory");
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    for (int kc = 0; kc < S && kc < nk; ++kc) load(kc);
  }
  __syncthreads();
  if (!(sched & SCHED_ACTOR)) {                                // critic-only step: drain the stages requested above, leave
    if (t == 0)
      for (int kc = 0; kc < S && kc < nk; ++kc) mbar_wait(full_bar(kc), 0u);
    return;
  }
  if (t == 0) TC_STAMP(1);

  const bool want_bsum = (P->mode == GEMM_WGRAD) && (P->C2 != nullptr) && (blockIdx.x == 0);
  float bs[4] = {0.f, 0.f, 0.f, 0.f};                         // bias-gradient partials: row m = t % 128, k rows 16 (t / 128) + 4 i + j
  float acc[NACC / 2], tot[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) tot[i] = 0.f;

  auto split = [&](int kc) {
    const int s = kc % S;
    mbar_wait(full_bar(s), (uint32_t)(kc / S) & 1u);
    uint8_t* st = gbase + (size_t)s * STAGE;
    if (want_bsum) {
      const float* rf = reinterpret_cast<const float*>(st) + (t >> 7) * 16 * TC_BM + (t & 127);
#pragma unroll
      for (int i = 0; i < 16; ++i) bs[i & 3] += rf[i * TC_BM];
    }
    tc_split<TC_BM>(st, st + HI_A, st + LO_A, a_mn, t);
    tc_split<BN>(st + RAW_B, st + HI_B, st + LO_B, b_mn, t);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma (async proxy)
    asm volatile("bar.sync 1, 256;" ::: "memory");            // both warpgroups' halves of the chunk are in place
  };

  split(0);
  for (int kc = 0;;) {
    {   // the 3 products x 4 k steps of 8 of chunk kc into a fresh accumulator
      const uint32_t st = base + (uint32_t)(kc % S) * STAGE;
      const uint64_t aH = wg_desc(st + HI_A + wg * 8192), aL = wg_desc(st + LO_A + wg * 8192);
      const uint64_t bH = wg_desc(st + HI_B), bL = wg_desc(st + LO_B);
      wg_fence_acc<NACC>(acc);
      wg_fence();
#pragma unroll
      for (int ks = 0; ks < TC_BK / 8; ++ks) {                 // k step of 8 tf32 = 32 B = 2 descriptor units
        if constexpr (PAIRED) {                                // bH spans [B_hi ; B_lo] as 2 BN rows
          // PTX orders accumulator accesses only between wgmma of the same shape: each of these two overlapping-register
          // MMAs of different N completes before the other shape is issued
          Wgmma<2 * BN>::mma(acc, aH + 2 * ks, bH + 2 * ks, ks > 0 ? 1u : 0u);
          wg_commit();
          wg_wait0();
          wg_fence_acc<NACC>(acc);
          wg_fence();
          Wgmma<BN>::mma(acc + BN / 2, aL + 2 * ks, bH + 2 * ks, 1u);
          wg_commit();
          wg_wait0();
          wg_fence_acc<NACC>(acc);
          wg_fence();
        } else {
          Wgmma<BN>::mma(acc, aH + 2 * ks, bH + 2 * ks, ks > 0 ? 1u : 0u);
          Wgmma<BN>::mma(acc, aH + 2 * ks, bL + 2 * ks, 1u);
          Wgmma<BN>::mma(acc, aL + 2 * ks, bH + 2 * ks, 1u);
        }
      }
      wg_commit();
      wg_fence_acc<NACC>(acc);
    }
    if (kc < 16 && t == 0) TC_STAMP(50 + 2 * kc);
    if (kc + 1 < nk) split(kc + 1);                           // overlaps the MMAs of chunk kc
    wg_wait0();
    wg_fence_acc<NACC>(acc);
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) tot[i] += PAIRED ? acc[i] + acc[BN / 2 + i] : acc[i];
    if ((t & 127) == 0) mbar_arrive(empty_bar(kc % S));
    if (t == 0 && kc + S < nk) {                               // refill the stage once the other warpgroup is done with it too
      mbar_wait(empty_bar(kc % S), (uint32_t)(kc / S) & 1u);
      load(kc + S);
    }
    if (kc < 16 && t == 0) TC_STAMP(51 + 2 * kc);
    if (++kc == nk) break;
  }
  if (t == 0) TC_STAMP(82);

  if (want_bsum) {       // 8 partials per column (4 per thread, two threads), summed in a fixed order: bit-reproducible
#pragma unroll
    for (int j = 0; j < 4; ++j) bsum_g[((t >> 7) * 4 + j) * TC_BM + (t & 127)] = bs[j];
    asm volatile("bar.sync 1, 256;" ::: "memory");
    const int m = m0 + t;
    if (t < TC_BM && m < M) {
      float ssum = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) ssum += bsum_g[r * TC_BM + t];
      P->C2[m] = ssum;
    }
  }

  // ---- epilogue: registers -> global ----
  const int mode = P->mode, relu = P->relu, ldc = P->ldc, ldmask = P->ldmask;
  const float* __restrict__ bias = P->bias;
  const float* __restrict__ mask = P->mask;
  float* __restrict__ Cout = P->C;
  const bool vec_c = ((ldc & 1) == 0) && ((reinterpret_cast<uintptr_t>(Cout) & 7) == 0);
  const int mrow = m0 + wg * 64 + ((t & 127) >> 5) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = n0 + 8 * j + 2 * (lane & 3);
    if (n >= N) continue;
    const bool two = n + 1 < N;
    float b0 = 0.f, b1 = 0.f;
    if (mode == GEMM_FWD && bias) { b0 = __ldg(bias + n); if (two) b1 = __ldg(bias + n + 1); }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = mrow + 8 * h;
      if (m >= M) continue;
      float x0 = tot[4 * j + 2 * h], x1 = tot[4 * j + 2 * h + 1];
      if (mode == GEMM_FWD) {
        x0 += b0; x1 += b1;
        if (relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
      } else if (mode == GEMM_DGRAD && mask) {
        const float* mp = mask + (long long)m * ldmask + n;
        if (!(ldg_f32(mp) > 0.f)) x0 = 0.f;
        if (two && !(ldg_f32(mp + 1) > 0.f)) x1 = 0.f;
      }
      float* cp = Cout + (long long)m * ldc + n;
      if (two && vec_c) {
        asm volatile("st.global.v2.f32 [%0], {%1, %2};" ::"l"(cp), "f"(x0), "f"(x1) : "memory");
      } else {
        stg_f32(cp, x0);
        if (two) stg_f32(cp + 1, x1);
      }
    }
  }
  if (t == 0) TC_STAMP(83);
}

}  // namespace bsac
