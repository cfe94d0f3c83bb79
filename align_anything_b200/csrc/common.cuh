// common.cuh -- shared device helpers for libaa_b200 (sm_90a only).
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/aa_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libaa_b200 is written for sm_90a (H100) only"
#endif

namespace aa {

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr int kWarp = 32;

// ---- host-side error plumbing (capi.cu) ------------------------------------------------
void set_error(const char *fmt, ...);
int check_launch(const char *what);  // cudaGetLastError -> 0 or positive code (+ message)
int sm_count();

#define AA_REQUIRE(cond, code, ...)     \
  do {                                  \
    if (!(cond)) {                      \
      ::aa::set_error(__VA_ARGS__);     \
      return (code);                    \
    }                                   \
  } while (0)

// ---- dtype traits -----------------------------------------------------------------------
template <typename T>
struct Traits;

template <>
struct Traits<__nv_bfloat16> {
  static constexpr int kCode = AA_BF16;
  static constexpr int kVec = 8;  // elements per 16-byte vector
  __device__ static __forceinline__ float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ static __forceinline__ __nv_bfloat16 from_float(float v) { return __float2bfloat16_rn(v); }
  __device__ static __forceinline__ float round(float v) {
    return __bfloat162float(__float2bfloat16_rn(v));
  }
};
template <>
struct Traits<__half> {
  static constexpr int kCode = AA_F16;
  static constexpr int kVec = 8;
  __device__ static __forceinline__ float to_float(__half v) { return __half2float(v); }
  __device__ static __forceinline__ __half from_float(float v) { return __float2half_rn(v); }
  __device__ static __forceinline__ float round(float v) { return __half2float(__float2half_rn(v)); }
};
template <>
struct Traits<float> {
  static constexpr int kCode = AA_F32;
  static constexpr int kVec = 4;
  __device__ static __forceinline__ float to_float(float v) { return v; }
  __device__ static __forceinline__ float from_float(float v) { return v; }
  __device__ static __forceinline__ float round(float v) { return v; }
};

// Round `v` to the precision of dtype code `dt` (bf16 / f16), identity for f32.
__device__ __forceinline__ float round_to(float v, int dt) {
  if (dt == AA_BF16) return __bfloat162float(__float2bfloat16_rn(v));
  if (dt == AA_F16) return __half2float(__float2half_rn(v));
  return v;
}

// Generic typed scalar load / store through a dtype code (cold paths: the PPO scalars).
__device__ __forceinline__ float load_as_float(const void *p, int64_t i, int dt) {
  if (dt == AA_BF16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16 *>(p)[i]);
  if (dt == AA_F16) return __half2float(reinterpret_cast<const __half *>(p)[i]);
  return reinterpret_cast<const float *>(p)[i];
}
__device__ __forceinline__ void store_from_float(void *p, int64_t i, int dt, float v) {
  if (dt == AA_BF16)
    reinterpret_cast<__nv_bfloat16 *>(p)[i] = __float2bfloat16_rn(v);
  else if (dt == AA_F16)
    reinterpret_cast<__half *>(p)[i] = __float2half_rn(v);
  else
    reinterpret_cast<float *>(p)[i] = v;
}
__host__ __device__ __forceinline__ int dtype_size(int dt) { return dt == AA_F32 ? 4 : 2; }

// ---- unpack one 32-bit word holding two 16-bit floats -----------------------------------
template <typename T>
__device__ __forceinline__ void unpack2(uint32_t w, float &lo, float &hi);
template <>
__device__ __forceinline__ void unpack2<__nv_bfloat16>(uint32_t w, float &lo, float &hi) {
  lo = __uint_as_float(w << 16);
  hi = __uint_as_float(w & 0xffff0000u);
}
template <>
__device__ __forceinline__ void unpack2<__half>(uint32_t w, float &lo, float &hi) {
  __half2 h = *reinterpret_cast<__half2 *>(&w);
  float2 f = __half22float2(h);
  lo = f.x;
  hi = f.y;
}
template <typename T>
__device__ __forceinline__ uint32_t pack2(float lo, float hi);
template <>
__device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);  // .x = lo (low 16 bits)
  return *reinterpret_cast<uint32_t *>(&h);
}
template <>
__device__ __forceinline__ uint32_t pack2<__half>(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t *>(&h);
}
// round two fp32 values to bf16 (RN-even) and back: ONE F2FP.PACK_AB + two ALU unpacks instead of two F2F on the
// quarter-rate XU pipe that the exp2 of the same epilogue needs
__device__ __forceinline__ void round_bf16_pair(float &a, float &b) {
  unpack2<__nv_bfloat16>(pack2<__nv_bfloat16>(a, b), a, b);
}

// ---- streaming 128-bit global access (read-once / write-once tiles) ---------------------
// loads: nc + L1::no_allocate + L2::256B prefetch
__device__ __forceinline__ uint4 ldg_stream(const uint4 *p) {
  uint4 r;
  asm("ld.global.nc.L1::no_allocate.L2::256B.v4.u32 {%0,%1,%2,%3}, [%4];"
      : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
      : "l"(p));
  return r;
}
// stores: .cs (evict-first)
__device__ __forceinline__ void stg_stream(uint4 *p, const uint4 &v) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// ---- fp32 pairs: the per-element math of the log-prob kernels is written two lanes at a time --------------
// sm_90 has no packed fp32 instructions, so each pair op is two scalar round-to-nearest ops.  The __f*_rn
// intrinsics are never contracted into FMAs, which the Veltkamp rounding below depends on.
typedef float2 f32x2;
__device__ __forceinline__ f32x2 f2_pack(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ void f2_unpack(f32x2 v, float &lo, float &hi) {
  lo = v.x;
  hi = v.y;
}
__device__ __forceinline__ f32x2 f2_splat(float v) { return f2_pack(v, v); }
__device__ __forceinline__ f32x2 f2_add(f32x2 a, f32x2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 f2_sub(f32x2 a, f32x2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 f2_mul(f32x2 a, f32x2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 f2_fma(f32x2 a, f32x2 b, f32x2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ f32x2 f2_ex2(f32x2 t) {
  float a, b;
  f2_unpack(t, a, b);
  return f2_pack(ex2_approx(a), ex2_approx(b));
}
// Round both lanes to 8 significant bits (= bf16 round-to-nearest) WITHOUT the conversion unit:
// Veltkamp splitting, hi = c - (c - x) with c = x * (2^16 + 1).  FMA-pipe ops instead of a conversion
// round trip, which shares its pipe with MUFU.EX2.
// Bit-identical to __float2bfloat16_rn for normal numbers (checked on 5M samples); inputs must be
// finite (callers clamp -inf logits to -1e30 first).
// `zero2` must be a RUN-TIME +0.0 pair (kernel parameter): ptxas may contract a multiply and a subtract
// into an FMA (d = fma(x, 65537, -x)), which destroys the split; producing c with an FMA whose addend
// the compiler cannot see through leaves nothing to contract.
__device__ __forceinline__ f32x2 f2_round_bf16(f32x2 x, f32x2 zero2) {
  const f32x2 c = f2_fma(x, f2_splat(65537.f), zero2);
  return f2_sub(c, f2_sub(c, x));
}
// Same for fp16 precision (11 significant bits): c = x * (2^13 + 1); valid inside fp16's normal range.
__device__ __forceinline__ f32x2 f2_round_f16(f32x2 x, f32x2 zero2) {
  const f32x2 c = f2_fma(x, f2_splat(8193.f), zero2);
  return f2_sub(c, f2_sub(c, x));
}

// ---- warp / block reductions ------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int warp_max_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Deterministic block sum (fixed tree); result valid in every thread.  `scratch` >= 33 floats.
template <int THREADS>
__device__ __forceinline__ float block_sum(float v, float *scratch) {
  constexpr int W = THREADS / kWarp;
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < kWarp) {
    float t = threadIdx.x < W ? scratch[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) scratch[32] = t;
  }
  __syncthreads();
  float r = scratch[32];
  __syncthreads();
  return r;
}

// Online-softmax partials are kept as (m, s) with s = sum_i 2^((x_i - m)*log2e).  The subtraction is
// done BEFORE the scaling (FADD + FMUL instead of one FFMA): x_i - m is exact for the element that
// attains the maximum, so its term is exactly 1 -- like ATen's exp(x - max) -- and a saturated row
// yields sum == 1.0f and a log-prob of exactly 0, which the multimodal PPO trainer's
// `response_mask = (log_probs != 0)` (trainers/text_image_to_text/ppo.py:250) depends on; it is also
// accurate for logits of any magnitude.
// Invariant: a partial whose max is -inf has s == 0.
__device__ __forceinline__ float lse_rescale(float m_old, float m_new) {
  if (m_old == m_new) return 1.f;
  if (m_old == -INFINITY) return 0.f;  // s == 0 anyway; avoids inf - inf
  return ex2_approx((m_old - m_new) * kLog2e);
}

// Merge two partials.
__device__ __forceinline__ void lse_merge(float &m, float &s, float m2, float s2) {
  const float mn = fmaxf(m, m2);
  s = s * lse_rescale(m, mn) + s2 * lse_rescale(m2, mn);
  m = mn;
}

// Fold one scalar element (the <8-element head / tail of an unaligned row).
__device__ __forceinline__ void lse_push(float &m, float &s, float x) {
  if (x == -INFINITY) return;  // exp(-inf) = 0: keeps the invariant
  lse_merge(m, s, x, 1.f);
}

// largest s in [0, n) with arr[s] <= key (arr ascending, arr[0] <= key)
__device__ __forceinline__ int upper_segment(const int64_t *__restrict__ arr, int n, int64_t key) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (__ldg(arr + mid) <= key)
      lo = mid;
    else
      hi = mid - 1;
  }
  return lo;
}

// "last block done" helper: returns true in every thread of the block that arrives last.
// `counter` must be zero before the first launch; the last block re-zeroes it.
__device__ __forceinline__ bool last_block_arrives(uint32_t *counter, uint32_t n_blocks) {
  __shared__ bool is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t prev = atomicAdd(counter, 1u);
    is_last = (prev == n_blocks - 1);
    if (is_last) *counter = 0u;
  }
  __syncthreads();
  if (is_last) __threadfence();
  return is_last;
}

// ---- one-shot all-reduce of a packed metric vector over NVLink peer memory -----------------------------
// Every rank owns one symmetric buffer (torch.distributed._symmetric_memory: peer-mapped over NVLink /
// NVSwitch) laid out as  float slots[2][world][kCollLanes]  followed by  uint32 flags[world].
// A call with epoch e: each rank STORES its n floats into slot [e & 1][rank] of EVERY peer's buffer
// (plain st.global on the peer-mapped pointer = NVLink write), fences system-wide, raises flag[rank] = e on
// every peer, waits until all `world` flags in its OWN buffer have reached e, then reduces the `world`
// slots locally (lanes in max_mask: MAX, others: mean -- the AVG / MAX of utils/multi_process.py:74-89).
// No NCCL launch, no extra kernel: it runs in the tail of the kernel that produced the vector (K2's last
// block, the PPO metric packer).  Double-buffered by epoch parity; epochs increase by 1 per call on
// every rank (same number of steps on every rank, as DistributedSampler guarantees).
constexpr int kCollLanes = 16;
struct CollParams {
  float *const *peer_bufs;  // device array [world] of peer-mapped buffer pointers (this rank's included)
  int rank, world;
  uint32_t epoch;
  uint32_t max_mask;        // bit t set: lane t is reduced with MAX instead of mean
};

__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Called by ONE block (>= 32 threads), all threads of its first warp; `vals` (local, n <= kCollLanes) in,
// reduced values out through `out`.
__device__ __forceinline__ void p2p_allreduce_packed(const CollParams &c, const float *vals, float *out, int n) {
  const int lane = threadIdx.x;
  if (lane >= kWarp) return;
  const int par = static_cast<int>(c.epoch & 1u);
  const size_t slot_floats = static_cast<size_t>(c.world) * kCollLanes;
  // 1. push my vector to every peer (lane t carries element t)
  if (lane < n) {
    const float v = vals[lane];
    for (int p = 0; p < c.world; ++p)
      c.peer_bufs[p][par * slot_floats + static_cast<size_t>(c.rank) * kCollLanes + lane] = v;
  }
  __threadfence_system();
  __syncwarp();
  // 2. raise my flag on every peer (lane p signals peer p)
  if (lane < c.world) {
    uint32_t *flags = reinterpret_cast<uint32_t *>(c.peer_bufs[lane] + 2 * slot_floats);
    st_release_sys(flags + c.rank, c.epoch);
  }
  // 3. wait for everybody's flag in MY buffer (lane p waits for rank p)
  float *mine = c.peer_bufs[c.rank];
  if (lane < c.world) {
    const uint32_t *flag = reinterpret_cast<const uint32_t *>(mine + 2 * slot_floats) + lane;
    while (static_cast<int32_t>(ld_acquire_sys(flag) - c.epoch) < 0) __nanosleep(64);
  }
  __syncwarp();
  // 4. reduce locally
  if (lane < n) {
    const volatile float *slots = mine + par * slot_floats;
    float acc = slots[lane];
    const bool is_max = (c.max_mask >> lane) & 1u;
    for (int r = 1; r < c.world; ++r) {
      const float v = slots[static_cast<size_t>(r) * kCollLanes + lane];
      acc = is_max ? fmaxf(acc, v) : acc + v;
    }
    out[lane] = is_max ? acc : acc / static_cast<float>(c.world);
  }
}

}  // namespace aa
