// Shared device/host helpers for the SAC learner kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bsac {

#define B200_HD __host__ __device__ __forceinline__
#define B200_D __device__ __forceinline__

constexpr int kWarp = 32;

// Schedule of the step in flight, one word per replica (Counters::sched), written by the ingest: SCHED_ACTOR = actor and
// temperature update, SCHED_TARGET = Polyak update of the targets.  A step without SCHED_ACTOR is a critic-only step.
enum { SCHED_ACTOR = 1, SCHED_TARGET = 2 };

// A replica's schedule word (null: a launch that always runs).  Every launch that reads it is at least two launches behind
// the ingest that wrote it on the same stream, or behind a full (event) dependency, so a kernel may read it BEFORE its
// griddepcontrol.wait, where the L2 round trip hides behind the wait instead of delaying the kernel: a kernel starts only
// after every CTA of the launch before it has exited, each of those passed its own griddepcontrol.wait, so the launch two
// back -- and every earlier one, the ingest included -- has completed and its writes are visible.  A kernel that skips its
// work still passes its own griddepcontrol.wait before it returns, which keeps that argument true for the launches after it.
// A full step must not wait for the word: kernels consume it where they wait for something else anyway.
// (__ldcg: an L2 load; nothing this SM cached can stand in for it.)
B200_D int sched_word(const int* sched) { return sched != nullptr ? __ldcg(sched) : SCHED_ACTOR | SCHED_TARGET; }

// ---------------------------------------------------------------------------------
// Philox4x32-10 counter-based generator (in-kernel noise + replay index sampling).
// ---------------------------------------------------------------------------------
struct Philox {
  uint32_t key[2];
  B200_HD Philox(uint64_t seed) {
    key[0] = (uint32_t)seed;
    key[1] = (uint32_t)(seed >> 32);
  }
  B200_HD static void mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
    uint64_t p = (uint64_t)a * b;
    hi = (uint32_t)(p >> 32);
    lo = (uint32_t)p;
  }
  // counter = (c0, c1, c2, c3) -> 4 x 32 random bits
  B200_HD void operator()(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t out[4]) const {
    uint32_t k0 = key[0], k1 = key[1];
#pragma unroll
    for (int r = 0; r < 10; ++r) {
      uint32_t hi0, lo0, hi1, lo1;
      mulhilo(0xD2511F53u, c0, hi0, lo0);
      mulhilo(0xCD9E8D57u, c2, hi1, lo1);
      uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
      c0 = n0; c1 = n1; c2 = n2; c3 = n3;
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
  }
};

B200_HD float u01(uint32_t x) {  // (0, 1]
  return ((float)(x >> 8) + 1.0f) * (1.0f / 16777216.0f);
}

// two independent N(0,1) from two 32-bit words (Box-Muller)
B200_D void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
  float u = u01(a), v = u01(b);
  float r = sqrtf(-2.0f * logf(u));
  float s, c;
  sincosf(6.28318530717958647692f * v, &s, &c);
  z0 = r * c;
  z1 = r * s;
}

// In-graph timeline: when enabled, the first thread of every kernel appends %globaltimer (ns) to a
// device buffer.  Kernels of a step run back to back on one stream, so consecutive differences are the
// true per-kernel times inside the CUDA graph (launch gaps included) -- unlike ncu's cold, serialised ones.
struct StampBuf { unsigned long long* t; int* idx; int cap; };
__device__ StampBuf g_stamp = {nullptr, nullptr, 0};
// Every step kernel starts with `KStamp ks_;`: (1) programmatic dependent launch -- the kernels are launched with
// programmatic stream serialization, so a kernel may be scheduled as soon as every CTA of its predecessor has exited
// (the implicit trigger) instead of after the predecessor's full completion + flush; griddepcontrol.wait then holds it
// until the predecessor's memory is visible.  No EARLY trigger (griddepcontrol.launch_dependents at entry): on the
// LunarLander step it lets the successor's CTAs crowd the SMs while the predecessor still runs, which was slower than
// no programmatic launch at all.  (2) the optional timeline stamp.  The stamp's enable
// pointer lives in global memory; loading it costs an L2 round trip, so thread 0 of CTA 0 only ISSUES the load at entry
// (with the entry time in a register) and consumes it in the destructor, i.e. when the kernel is done -- nothing on
// the critical path waits for it.
struct KStamp {
  unsigned long long t0;
  unsigned long long* buf;
  bool first;
  B200_D KStamp() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    first = (threadIdx.x | threadIdx.y | blockIdx.x | blockIdx.y | blockIdx.z) == 0;
    t0 = 0; buf = nullptr;
    if (first) {
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      buf = *(unsigned long long* volatile*)&g_stamp.t;
    }
  }
  B200_D ~KStamp() {
    if (first && buf != nullptr) {
      const int i = atomicAdd(g_stamp.idx, 1);
      if (i < g_stamp.cap) buf[i] = t0;
    }
  }
};

B200_D float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace bsac
