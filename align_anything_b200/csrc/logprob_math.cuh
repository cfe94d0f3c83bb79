// logprob_math.cuh -- device helpers shared by the log-prob kernels (logprob.cu: K1 / K1b; logprob_fused.cu: the
// single-pass forward + backward): packed online-softmax folds, the softmax-gradient math with the reference's
// rounding points, mbarrier / cp.async.bulk wrappers, the row-plan table.
#pragma once

#include "common.cuh"

namespace aa {

// Row plan (ops.RowPlan / ops.DevicePlan): per segment (one sample's scored run) the logits element offset, label
// offset, output offset and the prefix row count.
struct RowMap {
  const int64_t *seg_logit_off;
  const int64_t *seg_label_off;
  const int64_t *seg_out_off;
  const int64_t *seg_cum;
  int n_seg;
};

// ---- per-vector math ----------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float vec_max(const uint4 &v);

template <>
__device__ __forceinline__ float vec_max<__nv_bfloat16>(const uint4 &v) {
  // max is exact on the packed 16-bit values: 4 HMNMX2 instead of 8 FMNMX
  __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162 *>(&v.x);
  __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162 *>(&v.y);
  __nv_bfloat162 c = *reinterpret_cast<const __nv_bfloat162 *>(&v.z);
  __nv_bfloat162 d = *reinterpret_cast<const __nv_bfloat162 *>(&v.w);
  a = __hmax2(__hmax2(a, b), __hmax2(c, d));
  return fmaxf(__low2float(a), __high2float(a));
}
template <>
__device__ __forceinline__ float vec_max<__half>(const uint4 &v) {
  __half2 a = *reinterpret_cast<const __half2 *>(&v.x);
  __half2 b = *reinterpret_cast<const __half2 *>(&v.y);
  __half2 c = *reinterpret_cast<const __half2 *>(&v.z);
  __half2 d = *reinterpret_cast<const __half2 *>(&v.w);
  a = __hmax2(__hmax2(a, b), __hmax2(c, d));
  return fmaxf(__low2float(a), __high2float(a));
}
template <>
__device__ __forceinline__ float vec_max<float>(const uint4 &v) {
  return fmaxf(fmaxf(__uint_as_float(v.x), __uint_as_float(v.y)),
               fmaxf(__uint_as_float(v.z), __uint_as_float(v.w)));
}

// acc += 2^((x - mref)*log2e) for the 8 (or 4) elements of the vector, two lanes at a time (f32x2).
// Subtract first, then scale: x - m is exact for the maximum, so its term is exactly 1 (common.cuh).
template <typename T>
__device__ __forceinline__ void vec_expsum(const uint4 &v, f32x2 mref2, f32x2 L2, f32x2 &acc0, f32x2 &acc1) {
  if constexpr (sizeof(T) == 4) {
    acc0 = f2_add(acc0, f2_ex2(f2_mul(f2_sub(f2_pack(__uint_as_float(v.x), __uint_as_float(v.y)), mref2), L2)));
    acc1 = f2_add(acc1, f2_ex2(f2_mul(f2_sub(f2_pack(__uint_as_float(v.z), __uint_as_float(v.w)), mref2), L2)));
  } else {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float lo, hi;
      unpack2<T>(w[i], lo, hi);
      const f32x2 e = f2_ex2(f2_mul(f2_sub(f2_pack(lo, hi), mref2), L2));
      if (i & 1)
        acc1 = f2_add(acc1, e);
      else
        acc0 = f2_add(acc0, e);
    }
  }
}

// Fold a batch of N vectors into the running (m, s).
template <typename T, int N>
__device__ __forceinline__ void fold_batch(const uint4 (&v)[N], float &m, float &s, f32x2 L2) {
  float bm = vec_max<T>(v[0]);
#pragma unroll
  for (int u = 1; u < N; ++u) bm = fmaxf(bm, vec_max<T>(v[u]));
  const float mn = fmaxf(m, bm);
  const float mref = (mn == -INFINITY) ? 0.f : mn;  // everything so far is -inf: avoid inf - inf
  const f32x2 mref2 = f2_splat(mref);
  f32x2 acc0 = f2_pack(s * lse_rescale(m, mn), 0.f), acc1 = f2_pack(0.f, 0.f);
#pragma unroll
  for (int u = 0; u < N; ++u) vec_expsum<T>(v[u], mref2, L2, acc0, acc1);
  float a0, a1, a2, a3;
  f2_unpack(acc0, a0, a1);
  f2_unpack(acc1, a2, a3);
  s = (a0 + a1) + (a2 + a3);
  m = mn;
}

// ---- entropy: a third running sum next to (m, s) ----------------------------------------------------
// t = sum_j e^{x_j - m} (x_j - m) over the elements folded so far; the row's entropy is H = log s - t / s.  When the
// running maximum moves from m to m' (alpha = e^{m - m'}) the partial becomes t' = alpha (t + (m - m') s), the rule the
// fold, the thread merges and K6's split merge share.  A -inf logit adds 0 (the limit of p log p), an all -inf row has
// s = 0 and gets NaN.  The ENT = false forms below are the plain (m, s) code: t is dead and compiled away.
__device__ __forceinline__ float ent_rescale(float t, float s, float m_old, float m_new) {
  if (m_old == m_new) return t;
  if (m_old == -INFINITY) return 0.f;  // s == t == 0
  return lse_rescale(m_old, m_new) * fmaf(m_old - m_new, s, t);
}

template <bool ENT>
__device__ __forceinline__ void lse_merge_t(float &m, float &s, float &t, float m2, float s2, float t2) {
  if constexpr (ENT) {
    const float mn = fmaxf(m, m2);
    t = ent_rescale(t, s, m, mn) + ent_rescale(t2, s2, m2, mn);
    s = s * lse_rescale(m, mn) + s2 * lse_rescale(m2, mn);  // lse_merge's expression
    m = mn;
  } else {
    lse_merge(m, s, m2, s2);
  }
}

template <bool ENT>
__device__ __forceinline__ void lse_push_t(float &m, float &s, float &t, float x) {
  if constexpr (ENT) {
    if (x == -INFINITY) return;
    lse_merge_t<true>(m, s, t, x, 1.f, 0.f);
  } else {
    lse_push(m, s, x);
  }
}

// log s - t / s (fp32, never rounded)
__device__ __forceinline__ float entropy_of(float logsum, float s, float t) { return logsum - t / s; }

// vec_expsum plus tacc += e * (x - mref); the (x - mref) of a -inf logit is clamped so that its term is 0 * finite
template <typename T>
__device__ __forceinline__ void vec_expsum_ent(const uint4 &v, f32x2 mref2, f32x2 L2, f32x2 &acc0, f32x2 &acc1,
                                               f32x2 &tac0, f32x2 &tac1) {
  const f32x2 lim = f2_splat(-3.0e38f);
  auto term = [&](float lo, float hi, f32x2 &acc, f32x2 &tac) {
    const f32x2 d = f2_sub(f2_pack(lo, hi), mref2);
    const f32x2 e = f2_ex2(f2_mul(d, L2));
    acc = f2_add(acc, e);
    tac = f2_fma(e, make_float2(fmaxf(d.x, lim.x), fmaxf(d.y, lim.y)), tac);
  };
  if constexpr (sizeof(T) == 4) {
    term(__uint_as_float(v.x), __uint_as_float(v.y), acc0, tac0);
    term(__uint_as_float(v.z), __uint_as_float(v.w), acc1, tac1);
  } else {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float lo, hi;
      unpack2<T>(w[i], lo, hi);
      if (i & 1)
        term(lo, hi, acc1, tac1);
      else
        term(lo, hi, acc0, tac0);
    }
  }
}

// fold_batch, with the entropy sum when ENT
template <typename T, int N, bool ENT>
__device__ __forceinline__ void fold_batch_t(const uint4 (&v)[N], float &m, float &s, float &t, f32x2 L2) {
  if constexpr (ENT) {
    float bm = vec_max<T>(v[0]);
#pragma unroll
    for (int u = 1; u < N; ++u) bm = fmaxf(bm, vec_max<T>(v[u]));
    const float mn = fmaxf(m, bm);
    const float mref = (mn == -INFINITY) ? 0.f : mn;
    const f32x2 mref2 = f2_splat(mref);
    f32x2 acc0 = f2_pack(s * lse_rescale(m, mn), 0.f), acc1 = f2_pack(0.f, 0.f);
    f32x2 tac0 = f2_pack(ent_rescale(t, s, m, mn), 0.f), tac1 = f2_pack(0.f, 0.f);
#pragma unroll
    for (int u = 0; u < N; ++u) vec_expsum_ent<T>(v[u], mref2, L2, acc0, acc1, tac0, tac1);
    float a0, a1, a2, a3;
    f2_unpack(acc0, a0, a1);
    f2_unpack(acc1, a2, a3);
    s = (a0 + a1) + (a2 + a3);
    f2_unpack(tac0, a0, a1);
    f2_unpack(tac1, a2, a3);
    t = (a0 + a1) + (a2 + a3);
    m = mn;
  } else {
    fold_batch<T, N>(v, m, s, L2);
  }
}

// warp-level merge of (m, s[, t]) over all 32 lanes
template <bool ENT>
__device__ __forceinline__ void warp_lse_t(float &m, float &s, float &t) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
    const float s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const float t2 = ENT ? __shfl_xor_sync(0xffffffffu, t, o) : 0.f;
    lse_merge_t<ENT>(m, s, t, m2, s2, t2);
  }
}

template <int THREADS>
__device__ __forceinline__ void block_lse(float &m, float &s, float *sh_m, float *sh_s) {
  constexpr int NW = THREADS / kWarp;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float m2 = __shfl_xor_sync(0xffffffffu, m, o);
    float s2 = __shfl_xor_sync(0xffffffffu, s, o);
    lse_merge(m, s, m2, s2);
  }
  if (lane == 0) {
    sh_m[wid] = m;
    sh_s[wid] = s;
  }
  __syncthreads();
  if (wid == 0) {
    m = lane < NW ? sh_m[lane] : -INFINITY;
    s = lane < NW ? sh_s[lane] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float m2 = __shfl_xor_sync(0xffffffffu, m, o);
      float s2 = __shfl_xor_sync(0xffffffffu, s, o);
      lse_merge(m, s, m2, s2);
    }
  }
}

// block_lse, with the entropy sum when ENT (sh_t: 32 floats, unused otherwise)
template <int THREADS, bool ENT>
__device__ __forceinline__ void block_lse_t(float &m, float &s, float &t, float *sh_m, float *sh_s, float *sh_t) {
  if constexpr (ENT) {
    constexpr int NW = THREADS / kWarp;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    warp_lse_t<true>(m, s, t);
    if (lane == 0) {
      sh_m[wid] = m;
      sh_s[wid] = s;
      sh_t[wid] = t;
    }
    __syncthreads();
    if (wid == 0) {
      m = lane < NW ? sh_m[lane] : -INFINITY;
      s = lane < NW ? sh_s[lane] : 0.f;
      t = lane < NW ? sh_t[lane] : 0.f;
      warp_lse_t<true>(m, s, t);
    }
  } else {
    block_lse<THREADS>(m, s, sh_m, sh_s);
  }
}

// mbarrier / cp.async.bulk helpers (used by the bulk forward and the TMA-staged backward)
namespace bulk {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
template <typename T>
__device__ __forceinline__ uint4 neg_inf_vec() {
  if constexpr (sizeof(T) == 4) return make_uint4(0xff800000u, 0xff800000u, 0xff800000u, 0xff800000u);
  if constexpr (Traits<T>::kCode == AA_BF16) return make_uint4(0xff80ff80u, 0xff80ff80u, 0xff80ff80u, 0xff80ff80u);
  return make_uint4(0xfc00fc00u, 0xfc00fc00u, 0xfc00fc00u, 0xfc00fc00u);
}

}  // namespace bulk

// softmax probability of one element, the way the reference's backward sees it
template <typename T, bool FAITHFUL>
__device__ __forceinline__ float prob_of(float x, float m, float logsum, float c_f32) {
  if (FAITHFUL) {
    // ATen re-reads the ROUNDED log-softmax output: p = exp(round_T((x - max) - logsum))
    const float lp = Traits<T>::round((x - m) - logsum);
    return ex2_approx(lp * kLog2e);
  }
  return ex2_approx(fmaf(x, kLog2e, c_f32));
}

// Per-row constants of the backward, splatted once per row.
struct GradConsts {
  f32x2 m2, ls2, c2, ng2;  // max, logsum, -(max+logsum)*log2e, -g (times the offset residual in F32 mode)
  f32x2 zero2;             // run-time +0.0 (see f2_round_bf16)
};
__device__ __forceinline__ GradConsts make_grad_consts(float m, float logsum, float c_f32, float neg_g, float zero) {
  return GradConsts{f2_splat(m), f2_splat(logsum), f2_splat(c_f32), f2_splat(neg_g), f2_splat(zero)};
}

// -g * softmax for one pair of logits (f32x2).  FAITHFUL: p = exp(round_T((x - max) - logsum)), the value
// ATen's backward sees when it re-reads the ROUNDED log-softmax output; the rounding is done on the FMA
// pipe (Veltkamp split), not with a conversion round trip.
template <typename T, bool FAITHFUL>
__device__ __forceinline__ f32x2 pair_grad(f32x2 x2, const GradConsts &k) {
  f32x2 t;
  if (FAITHFUL) {
    f32x2 lp = f2_sub(f2_sub(x2, k.m2), k.ls2);
    lp = (Traits<T>::kCode == AA_BF16) ? f2_round_bf16(lp, k.zero2) : f2_round_f16(lp, k.zero2);
    t = f2_mul(lp, f2_splat(kLog2e));
  } else {
    t = f2_fma(x2, f2_splat(kLog2e), k.c2);
  }
  return f2_mul(f2_ex2(t), k.ng2);
}

template <typename T, bool FAITHFUL>
__device__ __forceinline__ uint4 vec_grad(const uint4 &v, const GradConsts &k) {
  uint4 r;
  if constexpr (sizeof(T) == 4) {
    float a, b, c, d;
    f2_unpack(pair_grad<T, FAITHFUL>(f2_pack(__uint_as_float(v.x), __uint_as_float(v.y)), k), a, b);
    f2_unpack(pair_grad<T, FAITHFUL>(f2_pack(__uint_as_float(v.z), __uint_as_float(v.w)), k), c, d);
    r = make_uint4(__float_as_uint(a), __float_as_uint(b), __float_as_uint(c), __float_as_uint(d));
  } else {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint32_t wi = w[i];
      if (FAITHFUL) {
        // -inf logits (masked vocabulary entries) would turn the Veltkamp split into inf - inf:
        // clamp them to a huge finite negative in the packed 16-bit domain (one HMNMX2 per pair)
        if constexpr (Traits<T>::kCode == AA_BF16) {
          const __nv_bfloat162 lim = __float2bfloat162_rn(-1e30f);
          __nv_bfloat162 h = __hmax2(*reinterpret_cast<__nv_bfloat162 *>(&wi), lim);
          wi = *reinterpret_cast<uint32_t *>(&h);
        } else {
          const __half2 lim = __float2half2_rn(-65504.f);
          __half2 h = __hmax2(*reinterpret_cast<__half2 *>(&wi), lim);
          wi = *reinterpret_cast<uint32_t *>(&h);
        }
      }
      float lo, hi;
      unpack2<T>(wi, lo, hi);
      f2_unpack(pair_grad<T, FAITHFUL>(f2_pack(lo, hi), k), lo, hi);
      o[i] = pack2<T>(lo, hi);
    }
    r = make_uint4(o[0], o[1], o[2], o[3]);
  }
  return r;
}

template <typename T, bool FAITHFUL>
__device__ __forceinline__ float grad_of(float x, float m, float logsum, float c_f32, float neg_g, float g, bool is_label) {
  const float pr = prob_of<T, FAITHFUL>(x, m, logsum, c_f32);
  if (is_label) return FAITHFUL ? __fsub_rn(g, __fmul_rn(pr, g)) : fmaf(pr, neg_g, g);
  return neg_g * pr;
}

// ---- entropy bonus: the entropy's gradient added to the gradient tile ---------------------------------------
// With l_k = x_k - m - logsum and p_k = e^{l_k}, dH/dx_k = -p_k (l_k + H), so a row whose entropy has the upstream
// gradient g_H gets  tile_k = [log-prob term] - g_H p_k (l_k + H).  p_k and l_k are the ones the log-prob term uses
// (FAITHFUL: the rounded log-softmax), the correction is fp32 and added before the tile's one rounding.  A -inf logit's
// l_k is clamped as in the entropy forward, so its term is e * finite = 0 before the coefficient multiplies it.
// Callers take these forms only for rows with g_H != 0: every other row runs the plain code and keeps its bits.
struct EntConsts {
  f32x2 h2, ngh2;  // H, -g_H (times the offset residual in F32 mode, like GradConsts::ng2)
};

template <typename T, bool FAITHFUL, bool PK>
__device__ __forceinline__ f32x2 pair_grad_ent(f32x2 x2, const GradConsts &k, const EntConsts &ek) {
  f32x2 lp = f2_sub(f2_sub(x2, k.m2), k.ls2), t;
  if (FAITHFUL) {
    if constexpr (PK && sizeof(T) == 2) {  // vec_grad_pk's rounding (logprob_fused.cu): one F2FP per pair, -inf stays -inf
      float lo, hi;
      f2_unpack(lp, lo, hi);
      unpack2<T>(pack2<T>(lo, hi), lo, hi);
      lp = f2_pack(lo, hi);
    } else {
      lp = (Traits<T>::kCode == AA_BF16) ? f2_round_bf16(lp, k.zero2) : f2_round_f16(lp, k.zero2);
    }
    t = f2_mul(lp, f2_splat(kLog2e));
  } else {
    t = f2_fma(x2, f2_splat(kLog2e), k.c2);
  }
  const f32x2 e = f2_ex2(t);
  const f32x2 d = f2_add(make_float2(fmaxf(lp.x, -3.0e38f), fmaxf(lp.y, -3.0e38f)), ek.h2);
  return f2_fma(f2_mul(e, d), ek.ngh2, f2_mul(e, k.ng2));
}

template <typename T, bool FAITHFUL, bool PK>
__device__ __forceinline__ uint4 vec_grad_ent(const uint4 &v, const GradConsts &k, const EntConsts &ek) {
  if constexpr (sizeof(T) == 4) {
    float a, b, c, d;
    f2_unpack(pair_grad_ent<T, FAITHFUL, PK>(f2_pack(__uint_as_float(v.x), __uint_as_float(v.y)), k, ek), a, b);
    f2_unpack(pair_grad_ent<T, FAITHFUL, PK>(f2_pack(__uint_as_float(v.z), __uint_as_float(v.w)), k, ek), c, d);
    return make_uint4(__float_as_uint(a), __float_as_uint(b), __float_as_uint(c), __float_as_uint(d));
  } else {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint32_t wi = w[i];
      if (FAITHFUL && !PK) {  // vec_grad's clamp: the Veltkamp split must not see -inf
        if constexpr (Traits<T>::kCode == AA_BF16) {
          const __nv_bfloat162 lim = __float2bfloat162_rn(-1e30f);
          __nv_bfloat162 h = __hmax2(*reinterpret_cast<__nv_bfloat162 *>(&wi), lim);
          wi = *reinterpret_cast<uint32_t *>(&h);
        } else {
          const __half2 lim = __float2half2_rn(-65504.f);
          __half2 h = __hmax2(*reinterpret_cast<__half2 *>(&wi), lim);
          wi = *reinterpret_cast<uint32_t *>(&h);
        }
      }
      float lo, hi;
      unpack2<T>(wi, lo, hi);
      f2_unpack(pair_grad_ent<T, FAITHFUL, PK>(f2_pack(lo, hi), k, ek), lo, hi);
      o[i] = pack2<T>(lo, hi);
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// the correction for one element (head / tail peel, element loops, the label column)
template <typename T, bool FAITHFUL>
__device__ __forceinline__ float ent_corr(float x, float m, float logsum, float c_f32, float ngh, float H) {
  float lp = (x - m) - logsum, e;
  if (FAITHFUL) {
    lp = Traits<T>::round(lp);
    e = ex2_approx(lp * kLog2e);
  } else {
    e = ex2_approx(fmaf(x, kLog2e, c_f32));
  }
  return (e * (fmaxf(lp, -3.0e38f) + H)) * ngh;
}

// grad_of, plus the entropy correction when `ent` (a row with g_H != 0)
template <typename T, bool FAITHFUL>
__device__ __forceinline__ float grad_of_ent(float x, float m, float logsum, float c_f32, float neg_g, float g,
                                             bool is_label, bool ent, float ngh, float H) {
  float v = grad_of<T, FAITHFUL>(x, m, logsum, c_f32, neg_g, g, is_label);
  if (ent) v += ent_corr<T, FAITHFUL>(x, m, logsum, c_f32, ngh, H);
  return v;
}

__device__ __forceinline__ uint32_t get_word(const uint4 &v, int i) {
  return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w));
}
__device__ __forceinline__ void set_word(uint4 &v, int i, uint32_t w) {
  if (i == 0) v.x = w; else if (i == 1) v.y = w; else if (i == 2) v.z = w; else v.w = w;
}

// Rewrite element k of the output vector with the one-hot (label) gradient; register-only
// (no dynamically indexed local arrays).
// ENT: the entropy correction is added when `ent` (see grad_of_ent); the ENT = false form is the plain code.
template <typename T, bool FAITHFUL, bool ENT = false>
__device__ __forceinline__ void patch_label(uint4 &o, const uint4 &in, int k, float m, float logsum, float c_f32,
                                            float neg_g, float g, bool ent = false, float ngh = 0.f, float H = 0.f) {
  if constexpr (sizeof(T) == 4) {
    const float x = __uint_as_float(get_word(in, k));
    const float gv = ENT ? grad_of_ent<T, FAITHFUL>(x, m, logsum, c_f32, neg_g, g, true, ent, ngh, H)
                         : grad_of<T, FAITHFUL>(x, m, logsum, c_f32, neg_g, g, true);
    set_word(o, k, __float_as_uint(gv));
  } else {
    const int w = k >> 1;
    const bool hi_half = (k & 1) != 0;
    float lo, hi;
    unpack2<T>(get_word(in, w), lo, hi);
    const float gv = ENT ? grad_of_ent<T, FAITHFUL>(hi_half ? hi : lo, m, logsum, c_f32, neg_g, g, true, ent, ngh, H)
                         : grad_of<T, FAITHFUL>(hi_half ? hi : lo, m, logsum, c_f32, neg_g, g, true);
    const uint32_t bits = pack2<T>(gv, gv) & 0xffffu;
    const uint32_t ow = get_word(o, w);
    set_word(o, w, hi_half ? ((ow & 0x0000ffffu) | (bits << 16)) : ((ow & 0xffff0000u) | bits));
  }
}

}  // namespace aa
