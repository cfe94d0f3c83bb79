// ppo.cu -- K4 / K5: PPO rollout-scoring scalars and losses.
//
// K4  aa_ppo_prep        : KL-shaped rewards (trainers/text_to_text/ppo.py:528-547), GAE reverse
//                          recurrence + returns (:487-508, a Python loop over t with ~5 kernels per
//                          step in the reference) and the row sums behind the metrics (:361-369).
// K5  aa_ppo_actor_loss  : clipped-ratio surrogate (:291-307) forward + backward in one launch.
//     aa_ppo_critic_loss : clipped value loss (:510-526) forward + backward in one launch.
//     aa_masked_mean     : utils/tools.py:460-467.
// K4r aa_ppo_returns     : Multi-PPO's reinforce / rloo / reinforce_baseline / group_norm returns
//                          (trainers/text_to_text/multi_ppo.py:510-591) on K4's shaped rewards.
//     aa_ppo_pack_metrics: the ten local scalars of :360-381 packed for ONE all-reduce.
//     aa_whiten_moments / aa_whiten_reduce / aa_whiten_apply: masked_whiten of a rollout's advantages.
//     aa_grpo_row_end, aa_entropy_hist_hi / _select_hi / _hist_lo / _select_lo: the exact entropy quantile of the
//                          top-entropy mask, and aa_grpo_loss_topent: GRPO's loss under that mask.
//     aa_cov_moments / _keys / _select_hi / _hist_lo / _select_lo / _mark: the exact top-k covariance selection of
//                          Clip-Cov and KL-Cov, and aa_ppo_actor_loss_cov / aa_grpo_loss_cov: the losses under it.
//     aa_ppo_actor_loss_pm / aa_grpo_loss_pm: the CISPO and SAPO policy losses (ppo_math.cuh, pm_token).
//
// These touch ~10 floats per token: latency-bound, not bandwidth-bound.  The point is launch
// count (thousands -> five) and zero host syncs; each sample is owned by one warp / CTA.
// "Rounding codes" reproduce the reference's eager per-op rounding when tensors are 16-bit.
#include "common.cuh"
#include "ppo_math.cuh"

namespace aa {

__device__ __forceinline__ int last_true(const uint8_t *mask_row, int W, int lane) {
  int end = -1;
  for (int base = W - 1; base >= 0 && end < 0; base -= kWarp) {
    const int pos = base - lane;
    const bool on = (pos >= 0) && mask_row[pos] != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, on);
    if (bal) end = base - (__ffs(bal) - 1);
  }
  return end;
}

// A_t = round(delta_t + round(cc * A_{t+1})) for t = hi .. lo, in place over sa[] (sa[t] holds delta_t on entry)
template <int DT>
__device__ __forceinline__ void gae_chain(float *sa, int hi, int lo, float cc) {
  float carry = 0.f;
  int t = hi;
  for (; t - 3 >= lo; t -= 4) {
    const float d0 = sa[t], d1 = sa[t - 1], d2 = sa[t - 2], d3 = sa[t - 3];
    const float a0 = round_to(d0 + round_to(cc * carry, DT), DT);
    const float a1 = round_to(d1 + round_to(cc * a0, DT), DT);
    const float a2 = round_to(d2 + round_to(cc * a1, DT), DT);
    const float a3 = round_to(d3 + round_to(cc * a2, DT), DT);
    sa[t] = a0; sa[t - 1] = a1; sa[t - 2] = a2; sa[t - 3] = a3;
    carry = a3;
  }
  for (; t >= lo; --t) {
    carry = round_to(sa[t] + round_to(cc * carry, DT), DT);
    sa[t] = carry;
  }
}

struct PrepParams {
  const void *lp, *ref_lp;
  int lp_dtype;
  int64_t lp_stride;
  const float *reward;
  const void *values;
  int val_dtype;
  int64_t val_stride;
  const uint8_t *mask;
  int64_t mask_stride;
  int B, W, start;
  float kl_coeff, clip, gamma, lam;
  int r_lp, r_v, r_a;  // rounding codes (AA_F32 = none)
  void *old_rewards;
  int rew_dtype;
  void *adv, *ret;
  int adv_dtype;
  float *row_stats;
  int32_t *status;
  int kl_est;  // the penalty's KL estimator (AA_KL_*; aa_ppo_prep: AA_KL_K1).  The metric row sums stay k1
};

// one warp per sample; the row (masked values, shaped rewards) is staged in shared memory so that the
// reverse recurrence never waits on global memory (2 x (W + 1) floats of dynamic shared memory)
__global__ void __launch_bounds__(32) ppo_prep_kernel(const PrepParams p) {
  extern __shared__ float sh[];
  const int b = blockIdx.x, lane = threadIdx.x;
  const int W = p.W, start = p.start, n = W - start;
  float *sv = sh;          // sv[t] = values[t] * mask[t], sv[W] = 0
  float *sr = sh + W + 1;  // sr[t] = rewards[t] * mask[t]
  float *sm = sr + W + 1;  // sm[t] = mask[t] as 0 / 1
  const uint8_t *mrow = p.mask + b * p.mask_stride;
  const int64_t lpo = b * p.lp_stride, vo = b * p.val_stride;
  const int64_t ro = static_cast<int64_t>(b) * W, ao = static_cast<int64_t>(b) * n;

  int end = last_true(mrow, W, lane);
  if (end < 0) {  // torch: m.nonzero()[-1] raises IndexError
    if (lane == 0 && p.status) atomicOr(p.status, AA_STATUS_EMPTY_MASK);
    end = 0;
  }
  const float rew_end = p.lp ? round_to(p.reward[b], p.r_lp) : 0.f;
  const float clip = round_to(p.clip, p.r_lp);

  // ---- KL-shaped, clipped per-token rewards + metric row sums ----
  // (p.lp == nullptr: `old_rewards` is an INPUT holding precomputed rewards -- GAE only)
  float kl_sum = 0.f, rkl_sum = 0.f, cnt = 0.f;
  for (int t = lane; t < W; t += kWarp) {
    const bool on = mrow[t] != 0;
    float kl = 0.f, r;
    if (p.lp) {
      const float x = load_as_float(p.lp, lpo + t, p.lp_dtype), rf = load_as_float(p.ref_lp, lpo + t, p.lp_dtype);
      float aux;
      kl = round_to(x - rf, p.r_lp);
      const float pen = (p.kl_est == AA_KL_K1) ? kl : kl_value(x, rf, p.kl_est, p.r_lp, aux);
      r = round_to(-p.kl_coeff * pen, p.r_lp);
      if (t == end) r = round_to(r + rew_end, p.r_lp);
      r = fminf(fmaxf(r, -clip), clip);
      store_from_float(p.old_rewards, ro + t, p.rew_dtype, r);
      r = round_to(r, p.rew_dtype);  // what a re-read of the stored tensor would give
    } else {
      r = load_as_float(p.old_rewards, ro + t, p.rew_dtype);
    }
    sr[t] = on ? r : 0.f;
    sv[t] = on ? load_as_float(p.values, vo + t, p.val_dtype) : 0.f;
    sm[t] = on ? 1.f : 0.f;
    if (t >= start && on) {
      kl_sum += kl;
      rkl_sum += r;
      cnt += 1.f;
    }
  }
  if (lane == 0) sv[W] = 0.f;
  kl_sum = round_to(warp_sum(kl_sum), p.r_lp);
  rkl_sum = round_to(warp_sum(rkl_sum), p.r_lp);
  cnt = warp_sum(cnt);
  __syncwarp();

  // ---- GAE: A_t = delta_t + gamma*lambda*A_{t+1}, t = W-1 .. start ----
  const float cc = p.gamma * p.lam;
  float adv_sum = 0.f, ret_sum = 0.f;
  auto delta_at = [&](int t) -> float {
    const float gv = round_to(p.gamma * sv[t + 1], p.r_v);
    const float a = round_to(sr[t] + gv, p.r_a);
    return round_to(a - sv[t], p.r_a);
  };
  const bool sequential = (p.r_a != AA_F32);
  if (sequential) {
    // 16-bit recurrence with the reference's rounding after every op: not associative, so the carry chain is
    // evaluated in order on one lane -- but ONLY the chain (2 flops + 2 roundings per step, out of shared
    // memory).  delta_t before it and returns / stores / metric sums after it run on all 32 lanes.  Beyond the
    // last attended position every term is +0, so the chain starts at `end`.
    for (int t = start + lane; t < W; t += kWarp) sr[t] = delta_at(t);  // sr[t] <- delta_t (own slot only)
    __syncwarp();
    if (lane == 0) {
      const int hi = (end < W - 1) ? end : W - 1;
      if (p.r_a == AA_BF16) gae_chain<AA_BF16>(sr, hi, start, cc);
      else gae_chain<AA_F16>(sr, hi, start, cc);
    }
    __syncwarp();
    for (int t = start + lane; t < W; t += kWarp) {
      const float a = sr[t];
      const float rt = round_to(a + sv[t], p.r_a);
      store_from_float(p.adv, ao + (t - start), p.adv_dtype, a);
      store_from_float(p.ret, ao + (t - start), p.adv_dtype, rt);
      adv_sum = fmaf(sm[t], a, adv_sum);
      ret_sum = fmaf(sm[t], rt, ret_sum);
    }
  } else {
    // fp32: warp-shuffle affine scan, 32 steps of the recurrence per pass
    float cpow = cc;  // cc^(lane+1)
    for (int k = 0; k < lane; ++k) cpow *= cc;
    float carry = 0.f;
    for (int i0 = 0; i0 < n; i0 += kWarp) {
      const int i = i0 + lane;
      const int t = W - 1 - i;
      float a = (i < n) ? delta_at(t) : 0.f;
      float pw = cc;
#pragma unroll
      for (int o = 1; o < kWarp; o <<= 1) {
        const float up = __shfl_up_sync(0xffffffffu, a, o);
        if (lane >= o) a = fmaf(pw, up, a);
        pw *= pw;
      }
      a = fmaf(cpow, carry, a);
      carry = __shfl_sync(0xffffffffu, a, kWarp - 1);
      if (i < n) {
        const float rt = a + sv[t];
        store_from_float(p.adv, ao + (t - start), p.adv_dtype, a);
        store_from_float(p.ret, ao + (t - start), p.adv_dtype, rt);
        adv_sum = fmaf(sm[t], a, adv_sum);
        ret_sum = fmaf(sm[t], rt, ret_sum);
      }
    }
  }
  adv_sum = warp_sum(adv_sum);
  ret_sum = warp_sum(ret_sum);
  if (lane == 0) {
    float *rs = p.row_stats + static_cast<int64_t>(b) * 8;
    rs[0] = kl_sum;
    rs[1] = rkl_sum;
    rs[2] = cnt;
    rs[3] = adv_sum / cnt;
    rs[4] = ret_sum / cnt;
    rs[5] = static_cast<float>(end);
    rs[6] = 0.f;
    rs[7] = 0.f;
  }
}

// ---- K4r: Multi-PPO returns (trainers/text_to_text/multi_ppo.py:510-591) ----------------------------------
// The four non-GAE estimators.  `rewards` is K4's (B, W) `old_rewards`; the reference masks it, applies the group
// statistic, then runs `cumulative_returns`, a Python loop over t with a float32 carry.  Group quirk (SURVEY H9): the
// estimators reshape the (B, W) TOKEN-reward matrix to (-1, n), so a group is n consecutive elements of the flattened
// tensor -- it may straddle rows, prompt positions take part, pad positions take part as zeros.
struct ReturnsParams {
  const void *rew;
  int rew_dtype;
  int64_t rew_stride;
  const uint8_t *mask;
  int64_t mask_stride;
  int B, W, start, est, n;
  float gamma;
  int r;         // rounding code: the rewards dtype (faithful) or AA_F32
  int mask_out;  // 1: outputs *= mask (get_advantages_and_returns); 0: cumulative_returns on its own
  void *adv, *ret;
  int out_dtype;
  float *row_stats;
};

// rewards * sequence_mask at flat index f of the (B, W) matrix (exact: r or a signed zero)
__device__ __forceinline__ float masked_reward(const ReturnsParams &p, int64_t f) {
  const int64_t b = f / p.W, t = f - b * p.W;
  const float r = load_as_float(p.rew, b * p.rew_stride + t, p.rew_dtype);
  return p.mask[b * p.mask_stride + t] ? r : r * 0.f;
}

// Welford state of ATen's std reduction (mean, m2, count)
struct Welford {
  float mean, m2, nf;
};
__device__ __forceinline__ Welford welford_one(float x) { return {x, 0.f, 1.f}; }
// WelfordOps::reduce (one element into a running state; {0, 0, 0} + x is exactly welford_one(x))
__device__ __forceinline__ Welford welford_add(Welford a, float x) {
  const float nf = __fadd_rn(a.nf, 1.f), d = __fsub_rn(x, a.mean), m = __fadd_rn(a.mean, __fdiv_rn(d, nf));
  return {m, __fmaf_rn(d, __fsub_rn(x, m), a.m2), nf};
}
// WelfordOps::combine of two non-empty states
__device__ __forceinline__ Welford welford_combine(Welford a, Welford b) {
  const float d = __fsub_rn(b.mean, a.mean), nn = __fadd_rn(a.nf, b.nf), r = __fdiv_rn(b.nf, nn);
  return {__fmaf_rn(d, r, a.mean), __fmaf_rn(__fmul_rn(__fmul_rn(d, d), a.nf), r, __fadd_rn(a.m2, b.m2)), nn};
}

// group_stats (below) for n >= 16
__device__ __forceinline__ void group_stats_wide(const ReturnsParams &p, int64_t g0, bool want_std, float &sum,
                                                 float &sd) {
  const int n = p.n;
  const int bw = n >= 32 ? 32 : 16;
  float ls[5], s = 0.f;  // ls[l]: the open subtree of 2^l partials
  Welford lw[5], w = {0.f, 0.f, 0.f};
#pragma unroll 1
  for (int j = 0; j < bw; ++j) {
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    Welford acc[2] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    for (int i = j; i < n; i += 4 * bw) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (i + q * bw < n) {
          const float x = masked_reward(p, g0 + i + q * bw);
          a[q] = __fadd_rn(a[q], x);
          if (want_std) acc[q & 1] = welford_add(acc[q & 1], x);
        }
      }
    }
    s = __fadd_rn(__fadd_rn(__fadd_rn(a[0], a[1]), a[2]), a[3]);
    if (want_std) w = acc[1].nf == 0.f ? acc[0] : welford_combine(acc[0], acc[1]);
    bool open = true;
#pragma unroll
    for (int l = 0; l < 5; ++l) {
      if (open && ((j >> l) & 1)) {
        s = __fadd_rn(ls[l], s);
        if (want_std) w = welford_combine(lw[l], w);
      } else if (open) {
        ls[l] = s;
        lw[l] = w;
        open = false;
      }
    }
  }
  sum = s;  // after partial bw - 1 (s, w): the whole tree
  sd = want_std ? __fsqrt_rn(__fdiv_rn(w.m2, static_cast<float>(n - 1))) : 0.f;
}

// Group sum and unbiased std of the n flat elements from g0, in the block-x layout Reduce.cuh describes for a
// contiguous inner dimension of n < 128 with at least 16 groups (larger n vectorises the loads, fewer groups widen
// the block past a warp): bw = min(largest power of two <= n, 32) threads; thread j folds elements j + k * bw, in k
// order, into accumulator k % 4 (the sum: vt0 = 4, from 0) or k % 2 (Welford: vt0 = 2), then combines its
// accumulators in index order; then a shuffle-down tree over the bw threads, lower index on the left.  The tree is
// evaluated here as a left-to-right pairwise fold over the threads' partials: partial j closes every subtree whose last
// leaf it is (one per trailing 1 bit of j), so ls / lw hold at most one open subtree per level.
// This is the layout as read, not confirmed at the bit level: on an H100 with torch 2.11, ATen's fp32 group sums equal
// it for n <= 3 only (for n = 4..8 they equal a 2-thread, 2-accumulator fold instead, and for n >= 12 no layout
// tried), so fp32 results match eager ATen on 75-90 % of the elements; 16-bit rounding hides the order (DESIGN
// section 4, "Multi-PPO (K4r)").  tests/test_gpu_returns_pin.py holds this order bit for bit against a float32
// restatement of it.
__device__ __forceinline__ void group_stats(const ReturnsParams &p, int64_t g0, bool want_std, float &sum, float &sd) {
  const int n = p.n;
  if (n < 16) {  // the same layout unrolled: bw <= 8 threads of at most two elements, a three-level tree
    const int bw = n >= 8 ? 8 : n >= 4 ? 4 : 2;
    float s[8];
    Welford w[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (j < bw) {
        const float a = masked_reward(p, g0 + j);
        const float b = (j + bw < n) ? masked_reward(p, g0 + j + bw) : 0.f;
        s[j] = (j + bw < n) ? __fadd_rn(a, b) : a;
        w[j] = (j + bw < n) ? welford_combine(welford_one(a), welford_one(b)) : welford_one(a);
      }
    }
#pragma unroll
    for (int off = 1; off < 8; off <<= 1) {
#pragma unroll
      for (int j = 0; j + off < 8; j += 2 * off) {
        if (j + off < bw) {
          s[j] = __fadd_rn(s[j], s[j + off]);
          if (want_std) w[j] = welford_combine(w[j], w[j + off]);
        }
      }
    }
    sum = s[0];
    sd = want_std ? __fsqrt_rn(__fdiv_rn(w[0].m2, static_cast<float>(n - 1))) : 0.f;
    return;
  }
  group_stats_wide(p, g0, want_std, sum, sd);
}

// the estimator's value at flat index f, with the rounding points of the eager ops (r = rounding code):
//   rloo               : r - round(round(round(sum) - r) * (1 / (n - 1)))   (ATen divides by a scalar via its reciprocal)
//   reinforce_baseline : r - round(sum * (1 / n))                           (the mean reduction's fp32 factor)
//   group_norm         : round(r - mean) / round(round(std) + 1e-9)         (std: unbiased, Welford in fp32)
__device__ __forceinline__ float estimator_value(const ReturnsParams &p, int64_t f) {
  const float x = masked_reward(p, f);
  if (p.est == AA_EST_REINFORCE) return x;
  const int n = p.n, rc = p.r;
  const int64_t g0 = (f / n) * n;
  float sum, sd;
  group_stats(p, g0, p.est == AA_EST_GROUP_NORM, sum, sd);
  if (p.est == AA_EST_GROUP_NORM) {
    const float mu = round_to(__fmul_rn(sum, __fdiv_rn(1.f, static_cast<float>(n))), rc);
    return round_to(__fdiv_rn(round_to(__fsub_rn(x, mu), rc), round_to(__fadd_rn(round_to(sd, rc), 1e-9f), rc)), rc);
  }
  if (p.est == AA_EST_RLOO) {
    const float loo = round_to(__fsub_rn(round_to(sum, rc), x), rc);
    const float base = round_to(__fmul_rn(loo, __fdiv_rn(1.f, static_cast<float>(n - 1))), rc);
    return round_to(__fsub_rn(x, base), rc);
  }
  const float mu = round_to(__fmul_rn(sum, __fdiv_rn(1.f, static_cast<float>(n))), rc);  // reinforce_baseline
  return round_to(__fsub_rn(x, mu), rc);
}

// one warp per sample: the estimator values of positions start..W-1 are staged in shared memory, the float32 carry
// c = r_t + gamma * c runs in order on one lane (one multiply, one add, each rounded: nothing contracts to an FMA), and
// all lanes store.  The chain runs over the whole response width: a masked position is `0 * value`, which is NaN where
// the estimator gave NaN (fp16 group_norm of a constant group: 1e-9 rounds to 0 in fp16), and that reaches every
// earlier return in the reference too.
__global__ void __launch_bounds__(32) ppo_returns_kernel(const ReturnsParams p) {
  extern __shared__ float sh[];
  const int b = blockIdx.x, lane = threadIdx.x;
  const int W = p.W, start = p.start, nr = W - start;
  const uint8_t *mrow = p.mask + b * p.mask_stride;
  const int64_t row0 = static_cast<int64_t>(b) * W, ao = static_cast<int64_t>(b) * nr;
  for (int t = start + lane; t < W; t += kWarp) {
    float v = estimator_value(p, row0 + t);
    if (!mrow[t]) v = v * 0.f;  // cumulative_returns masks again: `mask * rewards`
    sh[t - start] = v;
  }
  __syncwarp();
  if (lane == 0) {
    const float g = p.gamma;
    float c = 0.f;
    int t = nr - 1;
    for (; t >= 3; t -= 4) {
      const float r0 = sh[t], r1 = sh[t - 1], r2 = sh[t - 2], r3 = sh[t - 3];
      const float c0 = __fadd_rn(r0, __fmul_rn(g, c));
      const float c1 = __fadd_rn(r1, __fmul_rn(g, c0));
      const float c2 = __fadd_rn(r2, __fmul_rn(g, c1));
      c = __fadd_rn(r3, __fmul_rn(g, c2));
      sh[t] = round_to(c0, p.r); sh[t - 1] = round_to(c1, p.r); sh[t - 2] = round_to(c2, p.r); sh[t - 3] = round_to(c, p.r);
    }
    for (; t >= 0; --t) {
      c = __fadd_rn(sh[t], __fmul_rn(g, c));
      sh[t] = round_to(c, p.r);  // `returns[:, t] = cumulative_return` stores in the rewards dtype; the carry stays fp32
    }
  }
  __syncwarp();
  float sum = 0.f, cnt = 0.f;
  for (int t = start + lane; t < W; t += kWarp) {
    const bool on = mrow[t] != 0;
    const float v = (on || !p.mask_out) ? sh[t - start] : sh[t - start] * 0.f;  // `advantages *= mask`, `returns *= mask`
    store_from_float(p.adv, ao + (t - start), p.out_dtype, v);
    store_from_float(p.ret, ao + (t - start), p.out_dtype, v);
    if (on) {
      sum += v;
      cnt += 1.f;
    }
  }
  sum = warp_sum(sum);
  cnt = warp_sum(cnt);
  if (lane == 0 && p.row_stats) {  // K4's lanes 3 / 4: masked row means of advantages and returns
    float *rs = p.row_stats + static_cast<int64_t>(b) * 8;
    rs[3] = sum / cnt;
    rs[4] = sum / cnt;
  }
}

// ---- K5 ---------------------------------------------------------------------------------------
struct LossParams {
  const void *x;        // new log-probs / new values (the differentiable input)
  int64_t x_stride;
  const void *old;      // old log-probs / old values
  int64_t old_stride;
  int x_dtype;
  const void *aux;      // advantages / returns
  int64_t aux_stride;
  int aux_dtype;
  const uint8_t *mask;
  int64_t mask_stride;
  int B, Wm;
  float clip;
  int r_x, r_p;         // rounding codes: input dtype, promoted dtype
  float *loss;
  void *grad;
  int64_t grad_stride;
  float *row_mean;      // optional: masked row mean of x
  float *row_scratch;   // [B] per-row masked means of the objective
  uint32_t *counter;
  const int32_t *x_lens;  // optional: x[b, t] = t < R_b ? src[b, x_width - R_b + t] : 0, R_b = clamp(lens[b], 0, x_width)
  int x_width;            // (the pad_sequence of per-sample tails of text_image_to_text/ppo.py:318-330 folded into the load)
  // actor objective (aa_ppo_actor_loss_obj; aa_ppo_actor_loss: clip_hi = clip, dual = 0, agg = seq-mean-token-mean):
  // clip range [1 - clip, 1 + clip_hi], dual-clip factor (0 = off), `dual * adv` rounded to r_a, loss aggregation
  float clip_hi, dual;
  int r_a, agg;
  float *clip_frac;  // optional fp32[2]: clipped fraction, dual-clip fraction (row_scratch then holds 4 * B floats)
  // KL loss term (aa_ppo_actor_loss_kl; kl_coeff 0 = off): grad is d (loss + kl_coeff * agg(KL)) / d x, with the KL
  // of x against `ref` (x's dtype) by estimator kl_est; kl_loss[0] = agg(KL); row_scratch then holds 5 * B floats
  const void *ref;
  int64_t ref_stride;
  float kl_coeff;
  int kl_est;
  float *kl_loss;
  // Clip-Cov / KL-Cov (COV, aa_ppo_actor_loss_cov): the selection of aa_cov_mark (uint8, row stride sel_stride) and
  // KL-Cov's coefficient (cov_token)
  const uint8_t *sel;
  int64_t sel_stride;
  float cov_coef;
  // CISPO / SAPO (COV = AA_PM_*, aa_ppo_actor_loss_pm): SAPO's temperatures (pm_token); r_p is then s's dtype
  float tau_pos, tau_neg;
};

// COV (actor only): AA_COV_CLIP / AA_COV_KL (aa_ppo_actor_loss_cov), the token's objective is cov_token's;
// AA_PM_CISPO / AA_PM_SAPO (aa_ppo_actor_loss_pm), pm_token's
template <int THREADS, bool ACTOR, int COV = 0>
__global__ void __launch_bounds__(THREADS) ppo_loss_kernel(const LossParams p) {
  static_assert(ACTOR || COV == 0, "Clip-Cov and KL-Cov are actor objectives");
  __shared__ float scratch[33];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int Wm = p.Wm, rx = p.r_x, rp = p.r_p;
  const uint8_t *mrow = p.mask + b * p.mask_stride;
  const int64_t xo = b * p.x_stride, oo = b * p.old_stride, ao = b * p.aux_stride;

  const int x_rows = p.x_lens ? min(max(p.x_lens[b], 0), p.x_width) : Wm;
  const int x_shift = p.x_lens ? p.x_width - x_rows : 0;
  float cnt = 0.f;
  for (int t = tid; t < Wm; t += THREADS) cnt += mrow[t] ? 1.f : 0.f;
  cnt = block_sum<THREADS>(cnt, scratch);
  const bool token_mean = ACTOR && p.agg == AA_AGG_TOKEN_MEAN;
  float total = 0.f;  // token-mean: the micro-batch's masked-in token count (every block counts the whole mask)
  if (token_mean) {
    for (int k = 0; k < p.B; ++k)
      for (int t = tid; t < Wm; t += THREADS) total += p.mask[k * p.mask_stride + t] ? 1.f : 0.f;
    total = block_sum<THREADS>(total, scratch);
  }

  // upstream coefficient of d loss / d (row sum):  actor: -(1/B)/cnt (token-mean: -1/total) ; critic: 0.5*(1/B)/cnt.
  // Every count divides as the reference's int64 `mask.sum()` does: cast to the promoted dtype first (ppo_math.cuh)
  const float cnt_p = round_to(cnt, rp), total_p = round_to(total, rp);
  const float g_rs = ACTOR ? (token_mean ? actor_token_mean_coeff(total, rp) : actor_row_coeff(cnt, p.B, rp))
                           : round_to(round_to(round_to(0.5f, rp) / static_cast<float>(p.B), rp) / cnt_p, rp);
  const bool kl_on = ACTOR && p.kl_coeff != 0.f;
  const float g_kl = kl_on ? kl_term_coeff(p.kl_coeff, p.agg, token_mean ? total : cnt, p.B, rx) : 0.f;

  float row_sum = 0.f, x_sum = 0.f, kl_sum = 0.f;
  float n_clip = 0.f, n_dual = 0.f, n_neg = 0.f;  // clip-fraction counters of the row's masked-in tokens
  for (int t = tid; t < Wm; t += THREADS) {
    const bool on = mrow[t] != 0;
    const float x = (t < x_rows) ? load_as_float(p.x, xo + x_shift + t, p.x_dtype) : 0.f;
    const float old = load_as_float(p.old, oo + t, p.x_dtype);
    const float aux = load_as_float(p.aux, ao + t, p.aux_dtype);
    float obj, grad;
    if (ACTOR) {
      int why;
      if constexpr (COV == AA_PM_CISPO || COV == AA_PM_SAPO)
        pm_token(COV, x, old, aux, on, g_rs, p.clip_hi, p.tau_pos, p.tau_neg, rx, rp, obj, grad, why);
      else if constexpr (COV != 0)
        cov_token(COV, x, old, aux, on, on && p.sel[b * p.sel_stride + t] != 0, g_rs, p.clip, p.clip_hi, p.cov_coef,
                  rx, rp, obj, grad, why);
      else
        actor_token(x, old, aux, on, g_rs, p.clip, p.clip_hi, p.dual, rx, rp, p.r_a, obj, grad, why);
      if (on) {
        n_clip += (why & 1) ? 1.f : 0.f;
        n_dual += (why & 2) ? 1.f : 0.f;
        n_neg += (aux < 0.f) ? 1.f : 0.f;
      }
      if (kl_on && on) {  // the KL is created before the ratio: its gradient is added after the ratio's
        float kaux;
        kl_sum += kl_value(x, load_as_float(p.ref, b * p.ref_stride + t, p.x_dtype), p.kl_est, rx, kaux);
        grad = kl_grad(grad, g_kl, p.kl_est, kaux, rx);
      }
    } else {
      const float lo = round_to(old - p.clip, rx), hi = round_to(old + p.clip, rx);
      const float vc = fminf(fmaxf(x, lo), hi);
      const float d1 = round_to(x - aux, rp), d2 = round_to(vc - aux, rp);
      const float l1 = round_to(d1 * d1, rp), l2 = round_to(d2 * d2, rp);
      obj = fmaxf(l1, l2);
      if (l1 != l1 || l2 != l2) obj = NAN;
      const bool in_range = (x >= lo) && (x <= hi);
      float g1 = 0.f, g2 = 0.f;
      if (on) {
        if (l1 > l2) g1 = round_to(g_rs * (2.f * d1), rp);
        else if (l1 < l2) g2 = in_range ? round_to(g_rs * (2.f * d2), rp) : 0.f;
        else {  // a tie: maximum's backward sends round(grad / 2) down each branch
          const float half = round_to(0.5f * g_rs, rp);
          g1 = round_to(half * (2.f * d1), rp);
          g2 = in_range ? round_to(half * (2.f * d2), rp) : 0.f;
        }
      }
      grad = round_to(round_to(g1, rx) + round_to(g2, rx), rx);
    }
    if (on) {
      row_sum += round_to(obj, rp);
      x_sum += x;
    }
    if (p.grad) store_from_float(p.grad, b * p.grad_stride + t, p.x_dtype, on ? grad : 0.f);
  }
  row_sum = block_sum<THREADS>(row_sum, scratch);
  x_sum = block_sum<THREADS>(x_sum, scratch);
  const bool fracs = ACTOR && p.clip_frac;
  if (fracs) {
    n_clip = block_sum<THREADS>(n_clip, scratch);
    n_dual = block_sum<THREADS>(n_dual, scratch);
    n_neg = block_sum<THREADS>(n_neg, scratch);
  }
  if (kl_on) kl_sum = block_sum<THREADS>(kl_sum, scratch);
  if (tid == 0) {
    // seq-mean-token-mean: the row's masked mean in the promoted dtype; token-mean: the row's fp32 sum (rounded once,
    // after the cross-row sum, as ATen's sum over the whole tensor does).  The KL's rows alike, in the log-probs' dtype
    p.row_scratch[b] = token_mean ? row_sum : round_to(round_to(row_sum, rp) / cnt_p, rp);
    if (kl_on) p.row_scratch[4 * p.B + b] = token_mean ? kl_sum : round_to(round_to(kl_sum, rx) / round_to(cnt, rx), rx);
    if (p.row_mean) p.row_mean[b] = x_sum / cnt;
    if (fracs) {  // the counters reduced like the loss: per-row fractions (seq-mean) or raw counts (token-mean)
      const float d = token_mean ? 1.f : cnt;
      p.row_scratch[p.B + b] = n_clip / d;
      p.row_scratch[2 * p.B + b] = n_dual / d;
      p.row_scratch[3 * p.B + b] = n_neg / d;
    }
  }
  if (!last_block_arrives(p.counter, gridDim.x)) return;
  const volatile float *rows = p.row_scratch;
  float acc = 0.f;
  for (int k = tid; k < p.B; k += THREADS) acc += rows[k];
  acc = block_sum<THREADS>(acc, scratch);
  if (fracs) {
    float fc = 0.f, fd = 0.f, fn = 0.f;
    for (int k = tid; k < p.B; k += THREADS) {
      fc += rows[p.B + k];
      fd += rows[2 * p.B + k];
      fn += rows[3 * p.B + k];
    }
    fc = block_sum<THREADS>(fc, scratch);
    fd = block_sum<THREADS>(fd, scratch);
    fn = block_sum<THREADS>(fn, scratch);
    if (tid == 0) {
      // clipped: the masked mean of the indicator; dual: the share of negative-advantage tokens where c * adv wins
      // (the ratio of the two indicators' masked means; 0 without such tokens)
      p.clip_frac[0] = fc / (token_mean ? total : static_cast<float>(p.B));
      p.clip_frac[1] = fn > 0.f ? fd / fn : 0.f;
    }
  }
  if (kl_on) {
    float ak = 0.f;
    for (int k = tid; k < p.B; k += THREADS) ak += rows[4 * p.B + k];
    ak = block_sum<THREADS>(ak, scratch);
    if (tid == 0)
      p.kl_loss[0] = token_mean ? round_to(round_to(ak, rx) / round_to(total, rx), rx)
                                : round_to(ak / static_cast<float>(p.B), rx);
  }
  if (tid == 0) {
    const float mm = token_mean ? round_to(round_to(acc, rp) / total_p, rp) : round_to(acc / static_cast<float>(p.B), rp);
    const float loss = ACTOR ? -mm : round_to(0.5f * mm, rp);
    p.loss[0] = loss;
    // the same value as a 16-bit scalar in the first two bytes of loss[1]: the caller views it as the 0-dim bf16 / f16
    // tensor the reference's loss is, without a conversion launch
    if (rp != AA_F32) store_from_float(p.loss + 1, 0, rp, loss);
  }
}

// Gradient of the critic loss w.r.t. the RAW scores: the adjoint of `scores.squeeze(-1)[:, :-1]` followed by the
// pad_sequence of per-sample tails (text_image_to_text/ppo.py:318-330), times the upstream scalar -- one launch writes
// the whole (B, out_width) tile, zeros included.  The exact transpose of the critic's tail load (x_lens above): with
// R_b = clamp(lens[b], 0, src_width) and n_b = min(R_b, W),
//   out[b, t] = src_width - R_b <= t < src_width - R_b + n_b ? g * grad[b, t - (src_width - R_b)] : 0
template <typename T>
__global__ void __launch_bounds__(256)
    tail_scatter_scaled_kernel(const T *__restrict__ grad, int64_t grad_stride, const int32_t *__restrict__ lens, int W,
                               int src_width, const void *scale, int scale_dtype, T *__restrict__ out, int64_t out_stride,
                               int out_width) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= out_width) return;
  const int R = min(max(lens[b], 0), src_width);
  const int off = src_width - R, n = min(R, W);
  float v = 0.f;
  if (t >= off && t < off + n) {
    v = Traits<T>::to_float(grad[b * grad_stride + (t - off)]);
    if (scale) v = v * load_as_float(scale, 0, scale_dtype);  // fp32 product, one rounding (ATen's mul of a 16-bit tensor)
  }
  out[b * out_stride + t] = Traits<T>::from_float(v);
}


template <int THREADS>
__global__ void __launch_bounds__(THREADS)
    masked_mean_kernel(const void *x, int dtype, int64_t x_stride, const uint8_t *mask, int64_t mask_stride,
                       int B, int W, float *out, float *row_scratch, uint32_t *counter) {
  __shared__ float scratch[33];
  const int b = blockIdx.x, tid = threadIdx.x;
  float s = 0.f, c = 0.f;
  for (int t = tid; t < W; t += THREADS) {
    const bool on = mask ? mask[b * mask_stride + t] != 0 : true;
    if (on) {
      s += load_as_float(x, b * x_stride + t, dtype);
      c += 1.f;
    }
  }
  s = block_sum<THREADS>(s, scratch);
  c = block_sum<THREADS>(c, scratch);
  if (tid == 0) row_scratch[b] = mask ? s / c : s;
  if (!last_block_arrives(counter, gridDim.x)) return;
  const volatile float *rows = row_scratch;
  float acc = 0.f;
  for (int k = tid; k < B; k += THREADS) acc += rows[k];
  acc = block_sum<THREADS>(acc, scratch);
  if (tid == 0) out[0] = mask ? acc / static_cast<float>(B) : acc / (static_cast<float>(B) * static_cast<float>(W));
}

// ---- GRPO (SURVEY 8f row 2) -----------------------------------------------------------------------------
// trainers/text_to_text/grpo.py:268-318: group-normalised advantages, per-token KL (k3 estimator), per-token loss
// -(exp(lp - lp.detach()) * A - beta * KL), completion mask up to and including the first eos, loss = token mean.
__global__ void __launch_bounds__(32)
    group_advantages_kernel(const float *__restrict__ rewards, int n_groups, int G, float *__restrict__ adv) {
  // one warp per prompt group: mean, unbiased std (torch.std default), (r - mean) / (std + 1e-4)
  const int g = blockIdx.x, lane = threadIdx.x;
  if (g >= n_groups) return;
  float s = 0.f;
  for (int i = lane; i < G; i += kWarp) s += rewards[g * G + i];
  const float mean = warp_sum(s) / static_cast<float>(G);
  float q = 0.f;
  for (int i = lane; i < G; i += kWarp) {
    const float d = rewards[g * G + i] - mean;
    q += d * d;
  }
  const float sd = sqrtf(warp_sum(q) / static_cast<float>(G - 1)) + 1e-4f;
  for (int i = lane; i < G; i += kWarp) adv[g * G + i] = (rewards[g * G + i] - mean) / sd;
}

struct GrpoParams {
  const void *lp, *ref_lp;
  int dtype;
  int64_t lp_stride, ref_stride;
  const float *adv;
  const int32_t *row_end;
  const float *total;
  int B, K;
  float beta;
  int r_lp;  // rounding code
  float *loss;
  void *grad;
  int64_t grad_stride;
  float *row_scratch;
  uint32_t *counter;
};

// Dr. GRPO's advantages: r - group mean (the mean of group_advantages_kernel), no std scaling
__global__ void __launch_bounds__(32)
    group_centered_kernel(const float *__restrict__ rewards, int n_groups, int G, float *__restrict__ adv) {
  const int g = blockIdx.x, lane = threadIdx.x;
  if (g >= n_groups) return;
  float s = 0.f;
  for (int i = lane; i < G; i += kWarp) s += rewards[g * G + i];
  const float mean = warp_sum(s) / static_cast<float>(G);
  for (int i = lane; i < G; i += kWarp) adv[g * G + i] = rewards[g * G + i] - mean;
}

struct GrpoObjParams {
  GrpoParams base;
  const void *old;  // rollout-time policy log-probs, or nullptr: the log-probs themselves (ratio 1)
  int64_t old_stride;
  float clip_lo, clip_hi, dual;
  int agg;
  float *clip_frac;  // optional fp32[2]; row_scratch then holds 4 * B floats
  int kl_est;        // the per-token KL's estimator (AA_KL_*; aa_grpo_loss_obj: AA_KL_K3)
  // the top-entropy mask (TOPENT, aa_grpo_loss_topent): the policy's fp32 entropy (row stride ent_stride) and the
  // device threshold thr[0] of aa_entropy_select_lo; a counted token keeps s iff entropy >= thr
  const float *entropy;
  int64_t ent_stride;
  const float *thr;
  // Clip-Cov / KL-Cov (COV, aa_grpo_loss_cov): as LossParams' sel, sel_stride, cov_coef
  const uint8_t *sel;
  int64_t sel_stride;
  float cov_coef;
  // CISPO / SAPO (COV = AA_PM_*, aa_grpo_loss_pm): SAPO's temperatures
  float tau_pos, tau_neg;
};

// GRPO's loss and d loss / d lp, one block per row, the last block to arrive reduces the rows.  OBJECTIVE: the clipped
// objective (grpo_obj_token) under one of the three aggregations (aa_grpo_loss_obj); otherwise the reference's loss
// (grpo_token, aa_grpo_loss), which passes agg = token-mean, old = clip_frac = nullptr: g_t = 1 / total, the row
// partial is the fp32 row sum and the loss acc / total, as the reference computes them.  SEQUENCE (with OBJECTIVE,
// aa_grpo_loss_seq, old != nullptr): GSPO's sequence-level ratio -- the block first folds its row's summed log-ratio,
// then every token takes the row's objective and ratio coefficient (grpo_seq_row, grpo_seq_token).  TOPENT (with
// OBJECTIVE, aa_grpo_loss_topent): the top-entropy mask -- a counted token with entropy < thr keeps only its KL term
// (keep = 0 in grpo_obj_token; at sequence level s * keep, and s's gradient reaches the row's ratio from the kept
// tokens alone, n_s of grpo_seq_row).  COV (with OBJECTIVE at token level): Clip-Cov / KL-Cov (AA_COV_*,
// aa_grpo_loss_cov, grpo_cov_token) or CISPO / SAPO (AA_PM_*, aa_grpo_loss_pm, grpo_pm_token)
template <int THREADS, bool OBJECTIVE, bool SEQUENCE = false, bool TOPENT = false, int COV = 0>
__global__ void __launch_bounds__(THREADS) grpo_loss_kernel(const GrpoObjParams q) {
  static_assert(OBJECTIVE || !SEQUENCE, "the sequence-level ratio is an option of the clipped objective");
  static_assert(OBJECTIVE || !TOPENT, "the top-entropy mask is an option of the clipped objective");
  static_assert(COV == 0 || (OBJECTIVE && !SEQUENCE && !TOPENT), "Clip-Cov and KL-Cov are token-level objectives");
  __shared__ float scratch[33];
  const GrpoParams &p = q.base;
  const int b = blockIdx.x, tid = threadIdx.x, r = p.r_lp;
  const int end = p.row_end[b];
  const float total = p.total[0];
  const float A = p.adv[b];
  const float g_t = grpo_agg_coeff(q.agg, total, static_cast<float>(end), p.B, p.K);
  float thr = 0.f;
  if constexpr (TOPENT) thr = *q.thr;
  float row = 0.f, n_clip = 0.f, n_dual = 0.f;
  float s_seq = 0.f, coef_seq = 0.f;
  int why_seq = 0;
  if constexpr (SEQUENCE) {  // the masked-out tokens add (lp - old) * 0: nothing
    float lr = 0.f, kept = 0.f;
    for (int t = tid; t < end; t += THREADS) {
      lr += round_to(load_as_float(p.lp, b * p.lp_stride + t, p.dtype) -
                         load_as_float(q.old, b * q.old_stride + t, p.dtype),
                     r);
      if constexpr (TOPENT) kept += (q.entropy[b * q.ent_stride + t] >= thr) ? 1.f : 0.f;
    }
    const float S = round_to(block_sum<THREADS>(lr, scratch), r);
    float n_s = static_cast<float>(end);
    if constexpr (TOPENT) n_s = block_sum<THREADS>(kept, scratch);
    grpo_seq_row(S, static_cast<float>(end), n_s, A, g_t, q.clip_lo, q.clip_hi, q.dual, r, s_seq, coef_seq, why_seq);
  }
  for (int t = tid; t < p.K; t += THREADS) {
    const bool on = t < end;
    const float lp = load_as_float(p.lp, b * p.lp_stride + t, p.dtype);
    const float rf = load_as_float(p.ref_lp, b * p.ref_stride + t, p.dtype);
    float keep = 1.f;
    if constexpr (TOPENT) keep = (on && q.entropy[b * q.ent_stride + t] >= thr) ? 1.f : 0.f;
    float ptl, g;
    int why = 0;
    if constexpr (SEQUENCE) {
      grpo_seq_token(lp, rf, s_seq * keep, coef_seq, on, g_t, p.beta, q.kl_est, r, ptl, g);
      why = why_seq;
    } else if constexpr (COV == AA_PM_CISPO || COV == AA_PM_SAPO) {
      const float old = q.old ? load_as_float(q.old, b * q.old_stride + t, p.dtype) : lp;
      grpo_pm_token(COV, lp, old, rf, A, on, g_t, p.beta, q.clip_hi, q.tau_pos, q.tau_neg, q.kl_est, r, ptl, g, why);
    } else if constexpr (COV != 0) {
      const float old = q.old ? load_as_float(q.old, b * q.old_stride + t, p.dtype) : lp;
      grpo_cov_token(COV, lp, old, rf, A, on, on && q.sel[b * q.sel_stride + t] != 0, g_t, p.beta, q.clip_lo,
                     q.clip_hi, q.cov_coef, q.kl_est, r, ptl, g, why);
    } else if constexpr (OBJECTIVE) {
      const float old = q.old ? load_as_float(q.old, b * q.old_stride + t, p.dtype) : lp;
      grpo_obj_token(lp, old, rf, A, on, g_t, p.beta, q.clip_lo, q.clip_hi, q.dual, q.kl_est, r, ptl, g, why, keep);
    } else {
      grpo_token(lp, rf, A, on, g_t, p.beta, r, ptl, g);
    }
    if (on) {
      row += ptl;
      n_clip += (why & 1) ? 1.f : 0.f;
      n_dual += (why & 2) ? 1.f : 0.f;
    }
    if (p.grad) store_from_float(p.grad, b * p.grad_stride + t, p.dtype, g);
  }
  row = block_sum<THREADS>(row, scratch);
  const bool fracs = q.clip_frac != nullptr;
  if (fracs) {
    n_clip = block_sum<THREADS>(n_clip, scratch);
    n_dual = block_sum<THREADS>(n_dual, scratch);
  }
  const bool seq_mean = q.agg == AA_AGG_SEQ_MEAN_TOKEN_MEAN;
  if (tid == 0) {
    // seq-mean-token-mean: the row's token mean (the fp32 row sum over its count); otherwise the fp32 row sum
    p.row_scratch[b] = seq_mean ? row / static_cast<float>(end) : row;
    if (fracs) {  // per-row fractions (seq-mean-token-mean) or raw counts; the negative-advantage tokens are the row's
      const float d = seq_mean ? static_cast<float>(end) : 1.f;
      p.row_scratch[p.B + b] = n_clip / d;
      p.row_scratch[2 * p.B + b] = n_dual / d;
      p.row_scratch[3 * p.B + b] = (A < 0.f) ? static_cast<float>(end) / d : 0.f;
    }
  }
  if (!last_block_arrives(p.counter, gridDim.x)) return;
  const volatile float *rows = p.row_scratch;
  float acc = 0.f;
  for (int k = tid; k < p.B; k += THREADS) acc += rows[k];
  acc = block_sum<THREADS>(acc, scratch);
  if (fracs) {
    float fc = 0.f, fd = 0.f, fn = 0.f;
    for (int k = tid; k < p.B; k += THREADS) {
      fc += rows[p.B + k];
      fd += rows[2 * p.B + k];
      fn += rows[3 * p.B + k];
    }
    fc = block_sum<THREADS>(fc, scratch);
    fd = block_sum<THREADS>(fd, scratch);
    fn = block_sum<THREADS>(fn, scratch);
    if (tid == 0) {
      q.clip_frac[0] = fc / (seq_mean ? static_cast<float>(p.B) : total);
      q.clip_frac[1] = fn > 0.f ? fd / fn : 0.f;
    }
  }
  if (tid == 0) {
    if (q.agg == AA_AGG_SEQ_MEAN_TOKEN_SUM_NORM)
      p.loss[0] = acc / (static_cast<float>(p.B) * static_cast<float>(p.K));
    else
      p.loss[0] = seq_mean ? acc / static_cast<float>(p.B) : acc / total;
  }
}

// mean NLL over non-ignored rows (deterministic two-level reduction; last block finalises)
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
    nll_mean_kernel(const void *logp, int dtype, const int64_t *__restrict__ labels, int64_t n, int64_t ignore_index,
                    float *loss, float *neg_inv_count, float *partial, uint32_t *counter) {
  __shared__ float scratch[33];
  float s = 0.f, c = 0.f;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * THREADS + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * THREADS) {
    if (labels[i] != ignore_index) {
      s += load_as_float(logp, i, dtype);
      c += 1.f;
    }
  }
  s = block_sum<THREADS>(s, scratch);
  c = block_sum<THREADS>(c, scratch);
  if (threadIdx.x == 0) {
    partial[2 * blockIdx.x] = s;
    partial[2 * blockIdx.x + 1] = c;
  }
  if (!last_block_arrives(counter, gridDim.x)) return;
  const volatile float *pv = partial;
  float ts = 0.f, tc = 0.f;
  for (int k = threadIdx.x; k < static_cast<int>(gridDim.x); k += THREADS) {
    ts += pv[2 * k];
    tc += pv[2 * k + 1];
  }
  ts = block_sum<THREADS>(ts, scratch);
  tc = block_sum<THREADS>(tc, scratch);
  if (threadIdx.x == 0) {
    loss[0] = -ts / tc;            // all rows ignored -> 0/0 = NaN, like torch's mean over an empty set
    neg_inv_count[0] = -1.f / tc;
  }
}

__global__ void __launch_bounds__(32)
    ppo_pack_metrics_kernel(const float *__restrict__ row_stats, const float *__restrict__ reward,
                            const float *__restrict__ value_row_mean, const float *actor_loss,
                            const float *critic_loss, int B, float *stats, CollParams coll,
                            const int32_t *status) {
  const int lane = threadIdx.x;
  float kl = 0.f, rkl = 0.f, len = 0.f, adv = 0.f, ret = 0.f, rew = 0.f, val = 0.f, mx = 0.f;
  for (int b = lane; b < B; b += kWarp) {
    const float *rs = row_stats + static_cast<int64_t>(b) * 8;
    kl += rs[0];
    rkl += rs[1];
    len += rs[2];
    mx = fmaxf(mx, rs[2]);
    adv += rs[3];
    ret += rs[4];
    rew += reward[b];
    val += value_row_mean ? value_row_mean[b] : 0.f;
  }
  kl = warp_sum(kl); rkl = warp_sum(rkl); len = warp_sum(len); adv = warp_sum(adv);
  ret = warp_sum(ret); rew = warp_sum(rew); val = warp_sum(val); mx = warp_max(mx);
  if (lane == 0) {
    const float inv = 1.f / static_cast<float>(B);
    stats[0] = actor_loss ? actor_loss[0] : 0.f;
    stats[1] = critic_loss ? critic_loss[0] : 0.f;
    stats[2] = rew * inv;
    stats[3] = rkl * inv;
    stats[4] = adv * inv;
    stats[5] = ret * inv;
    stats[6] = val * inv;
    stats[7] = kl * inv;
    stats[8] = len * inv;
    stats[9] = mx;
    stats[10] = status ? static_cast<float>(*reinterpret_cast<const volatile int32_t *>(status)) : 0.f;  // MAX lane
    stats[11] = 0.f;
  }
  if (coll.world > 1) {  // the 9 x AVG + 1 x MAX all-reduces (+ barrier) of ppo.py:372-383, fused here
    __syncwarp();
    __threadfence();
    p2p_allreduce_packed(coll, stats, stats, 12);
  }
}

__global__ void __launch_bounds__(32) allreduce_packed_kernel(const float *src, float *dst, int n, CollParams coll) {
  p2p_allreduce_packed(coll, src, dst, n);
}

// ---- top-entropy token masking: the exact entropy quantile (TRL's top_entropy_quantile) ------------------------------
// thr = torch.quantile(H[counted], q) over every counted token of every rank, without a host sync: a radix select on
// order-preserving uint32 keys, 16 bits at a time.  aa_entropy_hist_hi counts the keys' high halves (and the NaNs),
// aa_entropy_select_hi finds the count N, the two ranks lo = floor(rank) and hi = ceil(rank) of rank = q * (N - 1) in
// fp32, and the high-half bucket of each; aa_entropy_hist_lo counts the low halves inside those one or two buckets and
// aa_entropy_select_lo reads the two values off and interpolates as ATen's lerp.  The histograms are integer counts, so
// the caller's all_reduce(SUM) between the passes gives every rank the same bits in any order.
constexpr int kEntBins = 1 << 16;         // bins of one 16-bit half
constexpr int kEntSelectThreads = 1024;   // one block scans the 2^16 bins, 64 per thread
constexpr uint32_t kEntSkip = 0xffffffffu;

// the float order as an unsigned order: -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf (NaNs are counted apart)
__device__ __forceinline__ uint32_t entropy_key(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float entropy_key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// sel[] of aa_entropy_select_hi: N, the NaN count, (bucket, rank inside it) of lo and of hi, and the weight's bits
enum { kSelN = 0, kSelNan, kSelLoBucket, kSelLoRank, kSelHiBucket, kSelHiRank, kSelWeight, kSelWords = 8 };

// HI: bin = the key's high half, or kEntBins for a NaN.  LO: the low half of a key whose high half is the lo bucket
// (bins [0, 2^16)) or else the hi bucket (bins [2^16, 2^17)); nothing when the select has no value to find.  One warp
// folds equal bins (__match_any_sync) into one integer atomic.  counted: t < row_end[b], or mask[b, t] != 0.
template <bool LO>
__global__ void __launch_bounds__(256)
    entropy_hist_kernel(const float *__restrict__ entropy, int64_t ent_stride, const int32_t *__restrict__ row_end,
                        const uint8_t *__restrict__ mask, int64_t mask_stride, int B, int K,
                        const uint32_t *__restrict__ sel, uint32_t *__restrict__ hist) {
  uint32_t lo_bucket = 0, hi_bucket = 0;
  if constexpr (LO) {
    if (sel[kSelN] == 0u || sel[kSelNan] != 0u) return;
    lo_bucket = sel[kSelLoBucket];
    hi_bucket = sel[kSelHiBucket];
  }
  const int64_t n = static_cast<int64_t>(B) * K;
  const int lane = threadIdx.x & (kWarp - 1);
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t base = static_cast<int64_t>(blockIdx.x) * blockDim.x + (threadIdx.x & ~(kWarp - 1)); base < n;
       base += stride) {
    const int64_t i = base + lane;
    uint32_t bin = kEntSkip;
    if (i < n) {
      const int b = static_cast<int>(i / K), t = static_cast<int>(i - static_cast<int64_t>(b) * K);
      const bool counted = mask ? mask[b * mask_stride + t] != 0 : t < row_end[b];
      if (counted) {
        const float h = entropy[b * ent_stride + t];
        if constexpr (!LO) {
          bin = (h != h) ? static_cast<uint32_t>(kEntBins) : entropy_key(h) >> 16;
        } else if (h == h) {
          const uint32_t k = entropy_key(h);
          if ((k >> 16) == lo_bucket)
            bin = k & 0xffffu;
          else if ((k >> 16) == hi_bucket)
            bin = kEntBins + (k & 0xffffu);
        }
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    if (bin != kEntSkip && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], static_cast<uint32_t>(__popc(peers)));
  }
}

// The whole block: the bin of h[0 .. 2^16) that holds rank r (0-based, r < the bins' sum) and r's rank inside it, to
// *bin / *rank_in (shared).  Also returns the bins' sum to every thread.
__device__ __forceinline__ uint32_t entropy_find_rank(const uint32_t *__restrict__ h, uint32_t r, uint32_t *bin, uint32_t *rank_in,
                                      uint32_t *warp_tot) {
  const int tid = threadIdx.x, lane = tid & (kWarp - 1), warp = tid >> 5;
  constexpr int per = kEntBins / kEntSelectThreads;
  const uint32_t *mine = h + tid * per;
  uint32_t s = 0;
#pragma unroll 8
  for (int j = 0; j < per; ++j) s += mine[j];
  uint32_t inc = s;  // inclusive scan: lanes, then warps
  for (int d = 1; d < kWarp; d <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += v;
  }
  __syncthreads();  // warp_tot may still be read by a previous call
  if (lane == kWarp - 1) warp_tot[warp] = inc;
  __syncthreads();
  uint32_t before = 0, all = 0;
#pragma unroll 4
  for (int w = 0; w < kEntSelectThreads / kWarp; ++w) {
    const uint32_t v = warp_tot[w];
    before += (w < warp) ? v : 0u;
    all += v;
  }
  const uint32_t excl = before + inc - s;
  if (r >= excl && r - excl < s) {
    uint32_t c = excl;
#pragma unroll 1
    for (int j = 0; j < per; ++j) {
      if (r - c < mine[j]) {
        *bin = static_cast<uint32_t>(tid * per + j);
        *rank_in = r - c;
        break;
      }
      c += mine[j];
    }
  }
  __syncthreads();
  return all;
}

// One block: N, the two ranks and their high-half buckets (sel[]).  rank = q * (N - 1) as ATen's quantile forms it
// (fp32 q times the count, rounded once), lo = floor(rank), hi = ceil(rank), both at most N - 1; weight = rank - lo.
__global__ void __launch_bounds__(kEntSelectThreads)
    entropy_select_hi_kernel(const uint32_t *__restrict__ hist, float q, uint32_t *__restrict__ sel) {
  __shared__ uint32_t warp_tot[kEntSelectThreads / kWarp];
  __shared__ uint32_t res[4];
  const int tid = threadIdx.x;
  const uint32_t N = entropy_find_rank(hist, 0xffffffffu, &res[0], &res[1], warp_tot);  // the sum alone
  if (N == 0u) {
    if (tid < kSelWords) sel[tid] = (tid == kSelNan) ? hist[kEntBins] : 0u;
    return;
  }
  const float rank = q * static_cast<float>(N - 1u);
  const double rk = static_cast<double>(rank);
  const uint32_t lo = rk >= static_cast<double>(N - 1u) ? N - 1u : static_cast<uint32_t>(rk);
  const double ce = ceil(rk);
  const uint32_t hi = ce >= static_cast<double>(N - 1u) ? N - 1u : static_cast<uint32_t>(ce);
  entropy_find_rank(hist, lo, &res[0], &res[1], warp_tot);
  entropy_find_rank(hist, hi, &res[2], &res[3], warp_tot);
  if (tid == 0) {
    sel[kSelN] = N;
    sel[kSelNan] = hist[kEntBins];
    sel[kSelLoBucket] = res[0];
    sel[kSelLoRank] = res[1];
    sel[kSelHiBucket] = res[2];
    sel[kSelHiRank] = res[3];
    sel[kSelWeight] = __float_as_uint(rank - static_cast<float>(lo));
    sel[7] = 0u;
  }
}

// One block: the two values and thr = lerp(v_lo, v_hi, w) as ATen's lerp forms it (w < 0.5: v_lo + w * (v_hi - v_lo),
// else v_hi - (v_hi - v_lo) * (1 - w), each a fused multiply-add); NaN when a counted entropy is NaN, and when nothing
// is counted (then no token is kept).
__global__ void __launch_bounds__(kEntSelectThreads)
    entropy_select_lo_kernel(const uint32_t *__restrict__ hist, const uint32_t *__restrict__ sel, float *thr) {
  __shared__ uint32_t warp_tot[kEntSelectThreads / kWarp];
  __shared__ uint32_t res[4];
  if (sel[kSelN] == 0u || sel[kSelNan] != 0u) {
    if (threadIdx.x == 0) thr[0] = __uint_as_float(0x7fc00000u);
    return;
  }
  const uint32_t lo_b = sel[kSelLoBucket], hi_b = sel[kSelHiBucket];
  entropy_find_rank(hist, sel[kSelLoRank], &res[0], &res[1], warp_tot);
  entropy_find_rank(hist + (hi_b == lo_b ? 0 : kEntBins), sel[kSelHiRank], &res[2], &res[3], warp_tot);
  if (threadIdx.x == 0) {
    const float v_lo = entropy_key_value((lo_b << 16) | res[0]);
    const float v_hi = entropy_key_value((hi_b << 16) | res[2]);
    const float w = __uint_as_float(sel[kSelWeight]);
    const float d = v_hi - v_lo;
    thr[0] = (fabsf(w) < 0.5f) ? fmaf(w, d, v_lo) : fmaf(-d, 1.f - w, v_hi);
  }
}

// ---- advantage whitening over a rollout (TRL's / verl's masked_whiten, shift_mean=True) -----------------------------
// The statistics are fp64 (n, sum A, sum A^2) triples.  Every sum has a fixed order, so a run reproduces its bits:
// each thread walks the same elements in the same order, then one fixed tree per block, then the K micro-batch slots
// in slot order.  There are no floating-point atomics.
constexpr int kWhitenThreads = 1024;

// Deterministic fp64 block sum (block_sum's fixed tree); result valid in every thread.  `scratch` >= 33 doubles.
template <int THREADS>
__device__ __forceinline__ double block_sum_f64(double v, double *scratch) {
  constexpr int W = THREADS / kWarp;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < kWarp) {
    double t = threadIdx.x < W ? scratch[threadIdx.x] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) scratch[32] = t;
  }
  __syncthreads();
  const double r = scratch[32];
  __syncthreads();
  return r;
}

// One CTA per micro-batch: a micro-batch's (B, W) advantages are a few thousand to a few hundred thousand elements, which
// one CTA reads in microseconds, so the sums need no cross-CTA combine (no partials, no counter).  The element loads are
// unconditional and masked by a select, so a masked-out NaN never enters the sums.
__global__ void __launch_bounds__(kWhitenThreads)
    whiten_moments_kernel(const void *adv, int dtype, int64_t adv_stride, const uint8_t *__restrict__ mask,
                          int64_t mask_stride, int B, int W, double *slot) {
  __shared__ double scratch[33];
  double n = 0.0, s1 = 0.0, s2 = 0.0;
  const uint32_t total = static_cast<uint32_t>(B) * static_cast<uint32_t>(W);  // < 2^31 (aa_whiten_moments)
#pragma unroll 4
  for (uint32_t i = threadIdx.x; i < total; i += kWhitenThreads) {
    const uint32_t b = i / static_cast<uint32_t>(W), t = i - b * static_cast<uint32_t>(W);
    const double a = load_as_float(adv, b * adv_stride + t, dtype);
    const bool on = mask[b * mask_stride + t] != 0;
    n += on ? 1.0 : 0.0;
    s1 += on ? a : 0.0;
    s2 += on ? a * a : 0.0;
  }
  n = block_sum_f64<kWhitenThreads>(n, scratch);
  s1 = block_sum_f64<kWhitenThreads>(s1, scratch);
  s2 = block_sum_f64<kWhitenThreads>(s2, scratch);
  if (threadIdx.x == 0) {
    slot[0] = n;
    slot[1] = s1;
    slot[2] = s2;
  }
}

// total[c] = sum over k = 0 .. K-1 of moments[k][c], in slot order (K is the rollout's micro-batch count)
__global__ void __launch_bounds__(32) whiten_reduce_kernel(const double *__restrict__ moments, int K, double *total) {
  const int c = threadIdx.x;
  if (c >= 3) return;
  double s = 0.0;
  for (int k = 0; k < K; ++k) s += moments[3 * k + c];
  total[c] = s;
}

// A' = (A - mean) * rstd where m, 0 where not m, in place.  mean and rstd = 1 / sqrt(var + 1e-8) (var unbiased, clamped at
// 0 against the rounding of sum A^2 - mean sum A) are formed in fp64 from the reduced triple and rounded once to fp32;
// the difference and the product are fp32, rounded once to the advantages' dtype.  n < 2 (masked_var's error) sets
// AA_STATUS_WHITEN_COUNT and writes nothing.
__global__ void __launch_bounds__(256)
    whiten_apply_kernel(void *adv, int dtype, int64_t adv_stride, const uint8_t *__restrict__ mask, int64_t mask_stride,
                        int W, const double *__restrict__ total, int32_t *status) {
  const int b = blockIdx.y;
  const int t = blockIdx.x * 256 + threadIdx.x;
  const double n = total[0];
  if (!(n >= 2.0)) {
    if (b == 0 && blockIdx.x == 0 && threadIdx.x == 0) atomicOr(status, AA_STATUS_WHITEN_COUNT);
    return;
  }
  if (t >= W) return;
  const double mean64 = total[1] / n;
  const double m2 = total[2] - total[1] * mean64;
  const double var = (m2 < 0.0 ? 0.0 : m2) / (n - 1.0);  // (a NaN stays NaN, as in masked_whiten)
  const float mean = static_cast<float>(mean64);
  const float rstd = static_cast<float>(1.0 / sqrt(var + 1e-8));
  const int64_t i = static_cast<int64_t>(b) * adv_stride + t;
  const bool on = mask[static_cast<int64_t>(b) * mask_stride + t] != 0;
  const float v = on ? __fmul_rn(__fsub_rn(load_as_float(adv, i, dtype), mean), rstd) : 0.f;
  store_from_float(adv, i, dtype, v);
}

// ---- Clip-Cov / KL-Cov: the exact top-k covariance selection (verl's clip_cov / kl_cov) -----------------------------
// The k largest uint32 keys of the eligible tokens of one loss call, without a host sync: the fp64 means (one block,
// fixed order), the keys with the high-half histogram, a radix select 16 bits a pass (entropy_find_rank on the
// threshold's ascending rank E - k), then a mark pass that takes the keys above the threshold T and, among the keys
// equal to T, the first `need` by flat index (a per-row tie count and an exclusive scan over the rows).
enum { kCovN = 0, kCovE, kCovK, kCovBucket, kCovRank, kCovT, kCovNeed, kCovMeanA, kCovMeanLp, kCovWords = 16 };
constexpr int kCovThreads = 256;

// MurmurHash3's 32-bit finaliser: a bijection of uint32
__host__ __device__ __forceinline__ uint32_t fmix32(uint32_t h) {
  h ^= h >> 16;
  h *= 0x85ebca6bu;
  h ^= h >> 13;
  h *= 0xc2b2ae35u;
  h ^= h >> 16;
  return h;
}

// the float order as an unsigned order, -0.0 folded onto +0.0 and every NaN above +inf (torch.topk's order)
__device__ __forceinline__ uint32_t cov_key(float x) {
  if (x != x) return 0xffffffffu;
  const uint32_t u = __float_as_uint(x == 0.f ? 0.f : x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// the counted tokens and their advantages: mask (B, W) with advantages (B, W) of adv_dtype, or row_end with fp32
// per-row advantages
struct CovRows {
  const void *lp;
  int64_t lp_stride;
  int lp_dtype;
  const void *adv;
  int64_t adv_stride;
  int adv_dtype;
  const uint8_t *mask;
  int64_t mask_stride;
  const int32_t *row_end;
  int B, W;
  __device__ __forceinline__ bool counted(int b, int t) const {
    return mask ? mask[b * mask_stride + t] != 0 : t < row_end[b];
  }
  __device__ __forceinline__ float advantage(int b, int t) const {
    return mask ? load_as_float(adv, b * adv_stride + t, adv_dtype) : static_cast<const float *>(adv)[b];
  }
};

// One block: (N, sum A, sum lp) in fp64, each thread over its elements in index order, then block_sum_f64's fixed
// tree; the loads are unconditional and masked by a select, so an uncounted NaN never enters the sums
__global__ void __launch_bounds__(kWhitenThreads) cov_moments_kernel(const CovRows c, uint32_t *state) {
  __shared__ double scratch[33];
  double n = 0.0, sa = 0.0, sl = 0.0;
  const uint32_t total = static_cast<uint32_t>(c.B) * static_cast<uint32_t>(c.W);
  for (uint32_t i = threadIdx.x; i < total; i += kWhitenThreads) {
    const int b = static_cast<int>(i / static_cast<uint32_t>(c.W)), t = static_cast<int>(i - b * static_cast<uint32_t>(c.W));
    const bool on = c.counted(b, t);
    const double a = c.advantage(b, t);
    const double l = load_as_float(c.lp, b * c.lp_stride + t, c.lp_dtype);
    n += on ? 1.0 : 0.0;
    sa += on ? a : 0.0;
    sl += on ? l : 0.0;
  }
  n = block_sum_f64<kWhitenThreads>(n, scratch);
  sa = block_sum_f64<kWhitenThreads>(sa, scratch);
  sl = block_sum_f64<kWhitenThreads>(sl, scratch);
  if (threadIdx.x == 0) {
    state[kCovN] = static_cast<uint32_t>(n);
    state[kCovMeanA] = __float_as_uint(static_cast<float>(sa / n));
    state[kCovMeanLp] = __float_as_uint(static_cast<float>(sl / n));
  }
}

struct CovKeyParams {
  CovRows c;
  const void *old;
  int64_t old_stride;
  float clip_lo, clip_hi, lb, ub;
  uint32_t seed;
  int rx, rp;
  const uint32_t *state;
  uint32_t *keys;
  uint8_t *elig;
  uint32_t *hist;
};

// keys, eligibility and the high-half histogram; one warp folds equal bins (__match_any_sync) into one atomic
template <int MODE>
__global__ void __launch_bounds__(kCovThreads) cov_keys_kernel(const CovKeyParams p) {
  const CovRows &c = p.c;
  const float mean_a = __uint_as_float(p.state[kCovMeanA]), mean_lp = __uint_as_float(p.state[kCovMeanLp]);
  const int64_t n = static_cast<int64_t>(c.B) * c.W;
  const int lane = threadIdx.x & (kWarp - 1);
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t base = static_cast<int64_t>(blockIdx.x) * blockDim.x + (threadIdx.x & ~(kWarp - 1)); base < n;
       base += stride) {
    const int64_t i = base + lane;
    uint32_t bin = kEntSkip;
    if (i < n) {
      const int b = static_cast<int>(i / c.W), t = static_cast<int>(i - static_cast<int64_t>(b) * c.W);
      const bool on = c.counted(b, t);
      const float a = c.advantage(b, t), lp = load_as_float(c.lp, b * c.lp_stride + t, c.lp_dtype);
      const float cov = __fmul_rn(__fsub_rn(a, mean_a), __fsub_rn(lp, mean_lp));
      bool e;
      uint32_t key;
      if constexpr (MODE == AA_COV_KL) {
        e = on;
        key = cov_key(cov);
      } else {
        const float old = p.old ? load_as_float(p.old, b * p.old_stride + t, c.lp_dtype) : lp;
        float obj, g;
        int why;
        actor_token(lp, old, a, false, 0.f, p.clip_lo, p.clip_hi, 0.f, p.rx, p.rp, p.rp, obj, g, why);
        e = on && !(why & 1) && cov > p.lb && cov < p.ub;
        key = fmix32(static_cast<uint32_t>(i) ^ p.seed);
      }
      p.keys[i] = key;
      p.elig[i] = e ? 1 : 0;
      if (e) bin = key >> 16;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    if (bin != kEntSkip && lane == __ffs(peers) - 1) atomicAdd(&p.hist[bin], static_cast<uint32_t>(__popc(peers)));
  }
}

// One block: E = the eligible count, k, and the bucket of ascending rank E - k (the k-th largest key)
__global__ void __launch_bounds__(kEntSelectThreads)
    cov_select_hi_kernel(const uint32_t *__restrict__ hist, double ratio, uint32_t *__restrict__ state) {
  __shared__ uint32_t warp_tot[kEntSelectThreads / kWarp];
  __shared__ uint32_t res[2];
  const uint32_t E = entropy_find_rank(hist, 0xffffffffu, &res[0], &res[1], warp_tot);  // the sum alone
  uint32_t k = 0;
  if (E > 0u) {
    const long long m = static_cast<long long>(ratio * static_cast<double>(state[kCovN]));  // Python's int()
    k = static_cast<uint32_t>(m < 1 ? 1 : (m > static_cast<long long>(E) ? static_cast<long long>(E) : m));
    entropy_find_rank(hist, E - k, &res[0], &res[1], warp_tot);
  }
  if (threadIdx.x == 0) {
    state[kCovE] = E;
    state[kCovK] = k;
    state[kCovBucket] = k ? res[0] : 0u;
    state[kCovRank] = k ? res[1] : 0u;
  }
}

__global__ void __launch_bounds__(kCovThreads)
    cov_hist_lo_kernel(const uint32_t *__restrict__ keys, const uint8_t *__restrict__ elig, int64_t n,
                       const uint32_t *__restrict__ state, uint32_t *__restrict__ hist) {
  if (state[kCovK] == 0u) return;
  const uint32_t bucket = state[kCovBucket];
  const int lane = threadIdx.x & (kWarp - 1);
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t base = static_cast<int64_t>(blockIdx.x) * blockDim.x + (threadIdx.x & ~(kWarp - 1)); base < n;
       base += stride) {
    const int64_t i = base + lane;
    uint32_t bin = kEntSkip;
    if (i < n && elig[i] && (keys[i] >> 16) == bucket) bin = keys[i] & 0xffffu;
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    if (bin != kEntSkip && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], static_cast<uint32_t>(__popc(peers)));
  }
}

// One block: the threshold key T and need = how many of the keys equal to T are selected; share = k / N
__global__ void __launch_bounds__(kEntSelectThreads)
    cov_select_lo_kernel(const uint32_t *__restrict__ hist, uint32_t *__restrict__ state, float *share) {
  __shared__ uint32_t warp_tot[kEntSelectThreads / kWarp];
  __shared__ uint32_t res[2];
  const uint32_t k = state[kCovK], N = state[kCovN];
  if (k == 0u) {
    if (threadIdx.x == 0) {
      state[kCovT] = 0xffffffffu;
      state[kCovNeed] = 0u;
      share[0] = 0.f;
    }
    return;
  }
  entropy_find_rank(hist, state[kCovRank], &res[0], &res[1], warp_tot);
  if (threadIdx.x == 0) {
    state[kCovT] = (state[kCovBucket] << 16) | res[0];
    state[kCovNeed] = hist[res[0]] - res[1];
    share[0] = static_cast<float>(static_cast<double>(k) / static_cast<double>(N));
  }
}

// Integer block sum (kCovThreads threads), valid in every thread; `scratch` >= kCovThreads / kWarp + 1 words
__device__ __forceinline__ uint32_t cov_block_sum(uint32_t v, uint32_t *scratch) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t s = 0;
#pragma unroll
  for (int w = 0; w < kCovThreads / kWarp; ++w) s += scratch[w];
  __syncthreads();
  return s;
}

// One block per row: the row's keys equal to T
__global__ void __launch_bounds__(kCovThreads)
    cov_tie_kernel(const uint32_t *__restrict__ keys, const uint8_t *__restrict__ elig, int W,
                   const uint32_t *__restrict__ state, int32_t *__restrict__ tie_rows) {
  __shared__ uint32_t scratch[kCovThreads / kWarp];
  const int b = blockIdx.x;
  const uint32_t T = state[kCovT];
  const int64_t row = static_cast<int64_t>(b) * W;
  uint32_t c = 0;
  if (state[kCovK] != 0u)
    for (int t = threadIdx.x; t < W; t += kCovThreads) c += (elig[row + t] && keys[row + t] == T) ? 1u : 0u;
  c = cov_block_sum(c, scratch);
  if (threadIdx.x == 0) tie_rows[b] = static_cast<int32_t>(c);
}

// One block per row: the ties of the rows before this one, then the row in chunks of kCovThreads, each tie's rank
// the exclusive scan of the tie bits in flat-index order
__global__ void __launch_bounds__(kCovThreads)
    cov_mark_kernel(const uint32_t *__restrict__ keys, const uint8_t *__restrict__ elig, int W,
                    const uint32_t *__restrict__ state, const int32_t *__restrict__ tie_rows, uint8_t *__restrict__ sel,
                    int64_t sel_stride) {
  __shared__ uint32_t scratch[kCovThreads / kWarp];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & (kWarp - 1), warp = tid >> 5;
  const uint32_t k = state[kCovK], T = state[kCovT], need = state[kCovNeed];
  const int64_t row = static_cast<int64_t>(b) * W;
  uint8_t *out = sel + static_cast<int64_t>(b) * sel_stride;
  if (k == 0u) {
    for (int t = tid; t < W; t += kCovThreads) out[t] = 0;
    return;
  }
  uint32_t before = 0;
  for (int j = tid; j < b; j += kCovThreads) before += static_cast<uint32_t>(tie_rows[j]);
  before = cov_block_sum(before, scratch);
  for (int t0 = 0; t0 < W; t0 += kCovThreads) {
    const int t = t0 + tid;
    const bool e = t < W && elig[row + t];
    const uint32_t key = e ? keys[row + t] : 0u;
    const bool tie = e && key == T;
    const unsigned bits = __ballot_sync(0xffffffffu, tie);
    if (lane == 0) scratch[warp] = __popc(bits);
    __syncthreads();
    uint32_t rank = before + __popc(bits & ((1u << lane) - 1u)), chunk = 0;
#pragma unroll
    for (int w = 0; w < kCovThreads / kWarp; ++w) {
      const uint32_t v = scratch[w];
      rank += (w < warp) ? v : 0u;
      chunk += v;
    }
    __syncthreads();
    if (t < W) out[t] = (e && (key > T || (tie && rank < need))) ? 1 : 0;
    before += chunk;
  }
}

static bool dtype_ok(int d) { return d == AA_BF16 || d == AA_F16 || d == AA_F32; }

}  // namespace aa

using namespace aa;

static int ppo_prep(const void *log_probs, const void *ref_log_probs, int lp_dtype, int64_t lp_row_stride,
                    const float *reward, const void *values, int val_dtype, int64_t val_row_stride, const uint8_t *mask,
                    int64_t mask_row_stride, int32_t B, int32_t W, int32_t start, float kl_coeff, int kl_estimator,
                    float clip_range_score, float gamma, float gae_lambda, int mode, void *old_rewards, int rew_dtype,
                    void *advantages, void *returns, int adv_dtype, float *row_stats, int32_t *status, void *stream) {
  AA_REQUIRE(B > 0 && W > 0 && start >= 0 && start < W, AA_ERR_ARG, "aa_ppo_prep: bad sizes (B=%d W=%d start=%d)", B, W, start);
  AA_REQUIRE(values && mask && old_rewards && advantages && returns && row_stats, AA_ERR_ARG,
             "aa_ppo_prep: null pointer");
  AA_REQUIRE((log_probs == nullptr) == (ref_log_probs == nullptr) && (log_probs == nullptr || reward != nullptr),
             AA_ERR_ARG, "aa_ppo_prep: log_probs, ref_log_probs and reward go together (all NULL = GAE only)");
  AA_REQUIRE(dtype_ok(lp_dtype) && dtype_ok(val_dtype) && dtype_ok(rew_dtype) && dtype_ok(adv_dtype), AA_ERR_DTYPE,
             "aa_ppo_prep: bad dtype");
  const bool f = (mode == AA_MODE_FAITHFUL);
  PrepParams p{log_probs, ref_log_probs, lp_dtype, lp_row_stride, reward, values, val_dtype, val_row_stride,
               mask, mask_row_stride, B, W, start, kl_coeff, clip_range_score, gamma, gae_lambda,
               f ? lp_dtype : AA_F32, f ? val_dtype : AA_F32, f ? adv_dtype : AA_F32,
               old_rewards, rew_dtype, advantages, returns, adv_dtype, row_stats, status, kl_estimator};
  const size_t smem = static_cast<size_t>(3 * (W + 1)) * sizeof(float);
  if (smem > 48 * 1024) {
    AA_REQUIRE(smem <= 200 * 1024, AA_ERR_UNSUPPORTED, "aa_ppo_prep: W=%d does not fit in shared memory", W);
    cudaError_t e = cudaFuncSetAttribute(ppo_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) {
      set_error("aa_ppo_prep: %s", cudaGetErrorString(e));
      return static_cast<int>(e);
    }
  }
  ppo_prep_kernel<<<B, 32, smem, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("aa_ppo_prep");
}

extern "C" int aa_ppo_prep(const void *log_probs, const void *ref_log_probs, int lp_dtype,
                           int64_t lp_row_stride, const float *reward, const void *values, int val_dtype,
                           int64_t val_row_stride, const uint8_t *mask, int64_t mask_row_stride, int32_t B,
                           int32_t W, int32_t start, float kl_coeff, float clip_range_score, float gamma,
                           float gae_lambda, int mode, void *old_rewards, int rew_dtype, void *advantages,
                           void *returns, int adv_dtype, float *row_stats, int32_t *status, void *stream) {
  return ppo_prep(log_probs, ref_log_probs, lp_dtype, lp_row_stride, reward, values, val_dtype, val_row_stride, mask,
                  mask_row_stride, B, W, start, kl_coeff, AA_KL_K1, clip_range_score, gamma, gae_lambda, mode,
                  old_rewards, rew_dtype, advantages, returns, adv_dtype, row_stats, status, stream);
}

extern "C" int aa_ppo_prep_kl(const void *log_probs, const void *ref_log_probs, int lp_dtype, int64_t lp_row_stride,
                              const float *reward, const void *values, int val_dtype, int64_t val_row_stride,
                              const uint8_t *mask, int64_t mask_row_stride, int32_t B, int32_t W, int32_t start,
                              float kl_coeff, int kl_estimator, float clip_range_score, float gamma, float gae_lambda,
                              int mode, void *old_rewards, int rew_dtype, void *advantages, void *returns,
                              int adv_dtype, float *row_stats, int32_t *status, void *stream) {
  AA_REQUIRE(kl_estimator_ok(kl_estimator), AA_ERR_ARG, "aa_ppo_prep_kl: unknown kl_estimator code %d", kl_estimator);
  AA_REQUIRE(isfinite(kl_coeff), AA_ERR_ARG, "aa_ppo_prep_kl: kl_coeff must be finite, got %g", kl_coeff);
  AA_REQUIRE(log_probs != nullptr, AA_ERR_ARG, "aa_ppo_prep_kl: log_probs is NULL (the GAE-only form is aa_ppo_prep)");
  return ppo_prep(log_probs, ref_log_probs, lp_dtype, lp_row_stride, reward, values, val_dtype, val_row_stride, mask,
                  mask_row_stride, B, W, start, kl_coeff, kl_estimator, clip_range_score, gamma, gae_lambda, mode,
                  old_rewards, rew_dtype, advantages, returns, adv_dtype, row_stats, status, stream);
}

extern "C" int aa_ppo_returns(const void *rewards, int rew_dtype, int64_t rew_row_stride, const uint8_t *mask,
                              int64_t mask_row_stride, int32_t B, int32_t W, int32_t start, int estimator,
                              int32_t n_samples_per_prompt, float gamma, int mode, int mask_outputs, void *advantages,
                              void *returns, int out_dtype, float *row_stats, void *stream) {
  AA_REQUIRE(B > 0 && W > 0 && start >= 0 && start < W, AA_ERR_ARG, "aa_ppo_returns: bad sizes (B=%d W=%d start=%d)", B,
             W, start);
  AA_REQUIRE(rewards && mask && advantages && returns && advantages != returns, AA_ERR_ARG,
             "aa_ppo_returns: null or aliased pointer");
  AA_REQUIRE(rew_row_stride >= W && mask_row_stride >= W, AA_ERR_ARG, "aa_ppo_returns: row strides must be >= W");
  AA_REQUIRE(estimator >= AA_EST_REINFORCE && estimator <= AA_EST_GROUP_NORM, AA_ERR_ARG,
             "aa_ppo_returns: unknown estimator code %d", estimator);
  const bool group = estimator != AA_EST_REINFORCE;
  AA_REQUIRE(n_samples_per_prompt >= (group ? 2 : 1), AA_ERR_ARG,
             "aa_ppo_returns: n_samples_per_prompt=%d (the group estimators need n > 1)", n_samples_per_prompt);
  AA_REQUIRE(!group || (static_cast<int64_t>(B) * W) % n_samples_per_prompt == 0, AA_ERR_ARG,
             "aa_ppo_returns: B*W=%lld is not a multiple of n_samples_per_prompt=%d",
             static_cast<long long>(B) * W, n_samples_per_prompt);
  AA_REQUIRE(dtype_ok(rew_dtype) && dtype_ok(out_dtype), AA_ERR_DTYPE, "aa_ppo_returns: bad dtype");
  const size_t smem = static_cast<size_t>(W - start) * sizeof(float);
  AA_REQUIRE(smem <= 200 * 1024, AA_ERR_UNSUPPORTED, "aa_ppo_returns: W - start = %d does not fit in shared memory",
             W - start);
  const bool f = (mode == AA_MODE_FAITHFUL);
  ReturnsParams p{rewards, rew_dtype, rew_row_stride, mask, mask_row_stride, B, W, start, estimator,
                  n_samples_per_prompt, gamma, f ? rew_dtype : AA_F32, mask_outputs != 0, advantages, returns, out_dtype,
                  row_stats};
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(ppo_returns_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) {
      set_error("aa_ppo_returns: %s", cudaGetErrorString(e));
      return static_cast<int>(e);
    }
  }
  ppo_returns_kernel<<<B, 32, smem, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("aa_ppo_returns");
}

static int promote(int a, int b) { return (a == b) ? a : AA_F32; }

static int ppo_actor_loss(const char *who, const void *log_probs, int64_t lp_stride, const void *old_log_probs,
                          int64_t old_stride, int lp_dtype, const void *advantages, int64_t adv_stride, int adv_dtype,
                          const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t Wm, float clip_low,
                          float clip_high, float dual_clip, int loss_agg, int mode, float *loss, void *grad,
                          int64_t grad_stride, float *clip_frac, float *row_scratch, uint32_t *counter, void *stream,
                          const void *ref = nullptr, int64_t ref_stride = 0, float kl_coeff = 0.f, int kl_est = 0,
                          float *kl_loss = nullptr) {
  AA_REQUIRE(B > 0 && Wm > 0, AA_ERR_ARG, "%s: bad sizes", who);
  AA_REQUIRE(log_probs && old_log_probs && advantages && mask && loss && row_scratch && counter, AA_ERR_ARG,
             "%s: null pointer", who);
  AA_REQUIRE(dtype_ok(lp_dtype) && dtype_ok(adv_dtype), AA_ERR_DTYPE, "%s: bad dtype", who);
  const bool f = (mode == AA_MODE_FAITHFUL);
  LossParams p{log_probs, lp_stride, old_log_probs, old_stride, lp_dtype, advantages, adv_stride, adv_dtype,
               mask, mask_stride, B, Wm, clip_low, f ? lp_dtype : AA_F32,
               f ? promote(lp_dtype, adv_dtype) : AA_F32, loss, grad, grad_stride, nullptr, row_scratch, counter, nullptr, 0,
               clip_high, dual_clip, f ? adv_dtype : AA_F32, loss_agg, clip_frac, ref, ref_stride, kl_coeff, kl_est,
               kl_loss};
  ppo_loss_kernel<128, true><<<B, 128, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch(who);
}

extern "C" int aa_ppo_actor_loss(const void *log_probs, int64_t lp_stride, const void *old_log_probs,
                                 int64_t old_stride, int lp_dtype, const void *advantages, int64_t adv_stride,
                                 int adv_dtype, const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t Wm,
                                 float clip_range_ratio, int mode, float *loss, void *grad, int64_t grad_stride,
                                 float *row_scratch, uint32_t *counter, void *stream) {
  return ppo_actor_loss("aa_ppo_actor_loss", log_probs, lp_stride, old_log_probs, old_stride, lp_dtype, advantages,
                        adv_stride, adv_dtype, mask, mask_stride, B, Wm, clip_range_ratio, clip_range_ratio, 0.f,
                        AA_AGG_SEQ_MEAN_TOKEN_MEAN, mode, loss, grad, grad_stride, nullptr, row_scratch, counter, stream);
}

extern "C" int aa_ppo_actor_loss_obj(const void *log_probs, int64_t lp_stride, const void *old_log_probs,
                                     int64_t old_stride, int lp_dtype, const void *advantages, int64_t adv_stride,
                                     int adv_dtype, const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t Wm,
                                     float clip_low, float clip_high, float dual_clip, int loss_agg, int mode,
                                     float *loss, void *grad, int64_t grad_stride, float *clip_frac, float *row_scratch,
                                     uint32_t *counter, void *stream) {
  AA_REQUIRE(actor_objective_ok(clip_low, clip_high, dual_clip, loss_agg), AA_ERR_ARG,
             "aa_ppo_actor_loss_obj: bad objective (need 0 <= clip_low < 1, clip_high >= 0, dual_clip 0 or > 1, a known "
             "loss_agg; got %g %g %g %d)", clip_low, clip_high, dual_clip, loss_agg);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "aa_ppo_actor_loss_obj: bad mode");
  return ppo_actor_loss("aa_ppo_actor_loss_obj", log_probs, lp_stride, old_log_probs, old_stride, lp_dtype, advantages,
                        adv_stride, adv_dtype, mask, mask_stride, B, Wm, clip_low, clip_high, dual_clip, loss_agg, mode,
                        loss, grad, grad_stride, clip_frac, row_scratch, counter, stream);
}

extern "C" int aa_ppo_actor_loss_kl(const void *log_probs, int64_t lp_stride, const void *old_log_probs,
                                    int64_t old_stride, int lp_dtype, const void *advantages, int64_t adv_stride,
                                    int adv_dtype, const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t Wm,
                                    float clip_low, float clip_high, float dual_clip, int loss_agg, int mode,
                                    const void *ref_log_probs, int64_t ref_stride, float kl_loss_coeff, int kl_estimator,
                                    float *loss, float *kl_loss, void *grad, int64_t grad_stride, float *clip_frac,
                                    float *row_scratch, uint32_t *counter, void *stream) {
  AA_REQUIRE(actor_objective_ok(clip_low, clip_high, dual_clip, loss_agg), AA_ERR_ARG,
             "aa_ppo_actor_loss_kl: bad objective (need 0 <= clip_low < 1, clip_high >= 0, dual_clip 0 or > 1, a known "
             "loss_agg; got %g %g %g %d)", clip_low, clip_high, dual_clip, loss_agg);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "aa_ppo_actor_loss_kl: bad mode");
  AA_REQUIRE(kl_estimator_ok(kl_estimator), AA_ERR_ARG, "aa_ppo_actor_loss_kl: unknown kl_estimator code %d",
             kl_estimator);
  AA_REQUIRE(kl_loss_term_ok(kl_loss_coeff), AA_ERR_ARG,
             "aa_ppo_actor_loss_kl: kl_loss_coeff must be finite and > 0 (got %g)", kl_loss_coeff);
  AA_REQUIRE(ref_log_probs && kl_loss, AA_ERR_ARG, "aa_ppo_actor_loss_kl: null ref_log_probs or kl_loss");
  return ppo_actor_loss("aa_ppo_actor_loss_kl", log_probs, lp_stride, old_log_probs, old_stride, lp_dtype, advantages,
                        adv_stride, adv_dtype, mask, mask_stride, B, Wm, clip_low, clip_high, dual_clip, loss_agg, mode,
                        loss, grad, grad_stride, clip_frac, row_scratch, counter, stream, ref_log_probs, ref_stride,
                        kl_loss_coeff, kl_estimator, kl_loss);
}

extern "C" int aa_ppo_critic_loss(const void *values, int64_t val_stride, const void *old_values,
                                  int64_t old_stride, int val_dtype, const void *returns, int64_t ret_stride,
                                  int ret_dtype, const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t Wm,
                                  float clip_range_value, int mode, float *loss, void *grad, int64_t grad_stride,
                                  float *row_mean, float *row_scratch, uint32_t *counter, const int32_t *value_tail_lens,
                                  int32_t value_src_width, void *stream) {
  AA_REQUIRE(B > 0 && Wm > 0, AA_ERR_ARG, "aa_ppo_critic_loss: bad sizes");
  AA_REQUIRE(!value_tail_lens || value_src_width > 0, AA_ERR_ARG, "aa_ppo_critic_loss: value_tail_lens needs value_src_width");
  AA_REQUIRE(values && old_values && returns && mask && loss && row_scratch && counter, AA_ERR_ARG,
             "aa_ppo_critic_loss: null pointer");
  AA_REQUIRE(dtype_ok(val_dtype) && dtype_ok(ret_dtype), AA_ERR_DTYPE, "aa_ppo_critic_loss: bad dtype");
  const bool f = (mode == AA_MODE_FAITHFUL);
  LossParams p{values, val_stride, old_values, old_stride, val_dtype, returns, ret_stride, ret_dtype,
               mask, mask_stride, B, Wm, clip_range_value, f ? val_dtype : AA_F32,
               f ? promote(val_dtype, ret_dtype) : AA_F32, loss, grad, grad_stride, row_mean, row_scratch, counter,
               value_tail_lens, value_src_width};
  ppo_loss_kernel<128, false><<<B, 128, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("aa_ppo_critic_loss");
}

extern "C" int aa_tail_scatter_scaled(const void *grad, int dtype, int64_t grad_row_stride, const int32_t *lens, int32_t B,
                                      int32_t W, int32_t src_width, const void *scale, int scale_dtype, void *out,
                                      int64_t out_row_stride, int32_t out_width, void *stream) {
  AA_REQUIRE(B > 0 && W > 0 && src_width > 0 && out_width >= src_width, AA_ERR_ARG, "aa_tail_scatter_scaled: bad sizes");
  AA_REQUIRE(grad && lens && out && grad != out, AA_ERR_ARG, "aa_tail_scatter_scaled: null or aliased pointers");
  AA_REQUIRE(dtype_ok(dtype) && (!scale || dtype_ok(scale_dtype)), AA_ERR_DTYPE, "aa_tail_scatter_scaled: bad dtype");
  const dim3 grid((out_width + 255) / 256, B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (dtype) {
    case AA_BF16:
      tail_scatter_scaled_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16 *>(grad), grad_row_stride, lens, W, src_width,
                                                                      scale, scale_dtype, static_cast<__nv_bfloat16 *>(out), out_row_stride, out_width);
      break;
    case AA_F16:
      tail_scatter_scaled_kernel<__half><<<grid, 256, 0, st>>>(static_cast<const __half *>(grad), grad_row_stride, lens, W, src_width, scale,
                                                               scale_dtype, static_cast<__half *>(out), out_row_stride, out_width);
      break;
    default:
      tail_scatter_scaled_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float *>(grad), grad_row_stride, lens, W, src_width, scale,
                                                              scale_dtype, static_cast<float *>(out), out_row_stride, out_width);
  }
  return check_launch("aa_tail_scatter_scaled");
}

extern "C" int aa_masked_mean(const void *x, int dtype, int64_t x_stride, const uint8_t *mask,
                              int64_t mask_stride, int32_t B, int32_t W, float *out, float *row_scratch,
                              uint32_t *counter, void *stream) {
  AA_REQUIRE(B > 0 && W > 0, AA_ERR_ARG, "aa_masked_mean: bad sizes");
  AA_REQUIRE(x && out && row_scratch && counter, AA_ERR_ARG, "aa_masked_mean: null pointer");
  AA_REQUIRE(dtype_ok(dtype), AA_ERR_DTYPE, "aa_masked_mean: bad dtype");
  masked_mean_kernel<128><<<B, 128, 0, static_cast<cudaStream_t>(stream)>>>(x, dtype, x_stride, mask, mask_stride,
                                                                               B, W, out, row_scratch, counter);
  return check_launch("aa_masked_mean");
}

extern "C" int aa_group_advantages(const float *rewards, int32_t n_groups, int32_t group_size, float *advantages,
                                   void *stream) {
  AA_REQUIRE(rewards && advantages && n_groups > 0 && group_size > 0, AA_ERR_ARG, "aa_group_advantages: bad arguments");
  group_advantages_kernel<<<n_groups, 32, 0, static_cast<cudaStream_t>(stream)>>>(rewards, n_groups, group_size, advantages);
  return check_launch("aa_group_advantages");
}

// aa_grpo_loss (objective false: the reference's loss, any mode), aa_grpo_loss_obj / _kl and aa_grpo_loss_seq
// (sequence: GSPO's sequence-level ratio, which needs the old log-probs): the checks, the completion mask (row_end, and
// the token count in scratch[0]) and the loss kernel over scratch + 1
static int grpo_loss(const char *who, bool objective, const void *log_probs, int64_t lp_stride, const void *ref_log_probs,
                     int64_t ref_stride, const void *old_log_probs, int64_t old_stride, int lp_dtype,
                     const float *advantages, const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id,
                     int32_t B, int32_t K, float beta, float clip_low, float clip_high, float dual_clip, int loss_agg,
                     int kl_estimator, int mode, float *loss, void *grad, int64_t grad_stride, float *clip_frac,
                     int32_t *row_end, float *scratch, uint32_t *counter, void *stream, bool sequence = false,
                     bool topent = false, const float *entropy = nullptr, int64_t ent_stride = 0,
                     const float *thr = nullptr, int cov = 0, float cov_coef = 0.f, const uint8_t *sel = nullptr,
                     int64_t sel_stride = 0, float tau_pos = 1.f, float tau_neg = 1.f) {
  AA_REQUIRE(B > 0 && K > 0 && log_probs && ref_log_probs && advantages && completion_tokens && loss && row_end &&
                 scratch && counter,
             AA_ERR_ARG, "%s: bad arguments", who);
  AA_REQUIRE(dtype_ok(lp_dtype), AA_ERR_DTYPE, "%s: bad dtype", who);
  AA_REQUIRE(!sequence || old_log_probs, AA_ERR_ARG,
             "%s: the sequence-level ratio needs old_log_probs (without them w = 1: use aa_grpo_loss_kl)", who);
  AA_REQUIRE(!topent || (entropy && thr && ent_stride >= K), AA_ERR_ARG,
             "%s: the top-entropy mask needs entropy (row stride >= K) and thr", who);
  if (objective) {
    AA_REQUIRE(grpo_objective_ok(clip_low, clip_high, dual_clip, loss_agg), AA_ERR_ARG,
               "%s: bad objective (need 0 <= clip_low < 1, clip_high >= 0, dual_clip 0 or > 1, a known loss_agg; got "
               "%g %g %g %d)", who, clip_low, clip_high, dual_clip, loss_agg);
    AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "%s: bad mode", who);
    AA_REQUIRE(kl_estimator_ok(kl_estimator), AA_ERR_ARG, "%s: unknown kl_estimator code %d", who, kl_estimator);
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  grpo_mask_kernel<128><<<B, 128, 0, st>>>(completion_tokens, tok_stride, B, K, eos_id, row_end, scratch, counter);
  int rc = check_launch(objective ? "aa_grpo_loss_obj(mask)" : "aa_grpo_loss(mask)");
  if (rc) return rc;
  GrpoObjParams q{GrpoParams{log_probs, ref_log_probs, lp_dtype, lp_stride, ref_stride, advantages, row_end, scratch, B,
                             K, beta, (mode == AA_MODE_FAITHFUL) ? lp_dtype : AA_F32, loss, grad, grad_stride,
                             scratch + 1, counter + 1},
                  old_log_probs, old_stride, clip_low, clip_high, dual_clip, loss_agg, clip_frac, kl_estimator,
                  entropy, ent_stride, thr, sel, sel_stride, cov_coef, tau_pos, tau_neg};
  if (cov == AA_PM_CISPO)
    grpo_loss_kernel<128, true, false, false, AA_PM_CISPO><<<B, 128, 0, st>>>(q);
  else if (cov == AA_PM_SAPO)
    grpo_loss_kernel<128, true, false, false, AA_PM_SAPO><<<B, 128, 0, st>>>(q);
  else if (cov == AA_COV_CLIP)
    grpo_loss_kernel<128, true, false, false, AA_COV_CLIP><<<B, 128, 0, st>>>(q);
  else if (cov == AA_COV_KL)
    grpo_loss_kernel<128, true, false, false, AA_COV_KL><<<B, 128, 0, st>>>(q);
  else if (topent && sequence)
    grpo_loss_kernel<128, true, true, true><<<B, 128, 0, st>>>(q);
  else if (topent)
    grpo_loss_kernel<128, true, false, true><<<B, 128, 0, st>>>(q);
  else if (sequence)
    grpo_loss_kernel<128, true, true><<<B, 128, 0, st>>>(q);
  else if (objective)
    grpo_loss_kernel<128, true><<<B, 128, 0, st>>>(q);
  else
    grpo_loss_kernel<128, false><<<B, 128, 0, st>>>(q);
  return check_launch(who);
}

extern "C" int aa_grpo_loss(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                            int lp_dtype, const float *advantages, const int64_t *completion_tokens,
                            int64_t tok_stride, int64_t eos_id, int32_t B, int32_t K, float beta, int mode,
                            float *loss, void *grad, int64_t grad_stride, int32_t *row_end, float *scratch,
                            uint32_t *counter, void *stream) {
  return grpo_loss("aa_grpo_loss", false, log_probs, lp_stride, ref_log_probs, ref_stride, nullptr, 0, lp_dtype,
                   advantages, completion_tokens, tok_stride, eos_id, B, K, beta, 0.f, 0.f, 0.f, AA_AGG_TOKEN_MEAN,
                   AA_KL_K3, mode, loss, grad, grad_stride, nullptr, row_end, scratch, counter, stream);
}

extern "C" int aa_group_advantages_centered(const float *rewards, int32_t n_groups, int32_t group_size,
                                            float *advantages, void *stream) {
  AA_REQUIRE(rewards && advantages && n_groups > 0 && group_size > 0, AA_ERR_ARG,
             "aa_group_advantages_centered: bad arguments");
  group_centered_kernel<<<n_groups, 32, 0, static_cast<cudaStream_t>(stream)>>>(rewards, n_groups, group_size,
                                                                                advantages);
  return check_launch("aa_group_advantages_centered");
}

extern "C" int aa_grpo_loss_obj(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                                const void *old_log_probs, int64_t old_stride, int lp_dtype, const float *advantages,
                                const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B,
                                int32_t K, float beta, float clip_low, float clip_high, float dual_clip, int loss_agg,
                                int mode, float *loss, void *grad, int64_t grad_stride, float *clip_frac,
                                int32_t *row_end, float *scratch, uint32_t *counter, void *stream) {
  return grpo_loss("aa_grpo_loss_obj", true, log_probs, lp_stride, ref_log_probs, ref_stride, old_log_probs, old_stride,
                   lp_dtype, advantages, completion_tokens, tok_stride, eos_id, B, K, beta, clip_low, clip_high,
                   dual_clip, loss_agg, AA_KL_K3, mode, loss, grad, grad_stride, clip_frac, row_end, scratch, counter,
                   stream);
}

extern "C" int aa_grpo_loss_kl(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                               const void *old_log_probs, int64_t old_stride, int lp_dtype, const float *advantages,
                               const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B,
                               int32_t K, float beta, float clip_low, float clip_high, float dual_clip, int loss_agg,
                               int kl_estimator, int mode, float *loss, void *grad, int64_t grad_stride,
                               float *clip_frac, int32_t *row_end, float *scratch, uint32_t *counter, void *stream) {
  return grpo_loss("aa_grpo_loss_kl", true, log_probs, lp_stride, ref_log_probs, ref_stride, old_log_probs, old_stride,
                   lp_dtype, advantages, completion_tokens, tok_stride, eos_id, B, K, beta, clip_low, clip_high,
                   dual_clip, loss_agg, kl_estimator, mode, loss, grad, grad_stride, clip_frac, row_end, scratch,
                   counter, stream);
}

extern "C" int aa_grpo_loss_seq(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                                const void *old_log_probs, int64_t old_stride, int lp_dtype, const float *advantages,
                                const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B,
                                int32_t K, float beta, float clip_low, float clip_high, float dual_clip, int loss_agg,
                                int kl_estimator, int mode, float *loss, void *grad, int64_t grad_stride,
                                float *clip_frac, int32_t *row_end, float *scratch, uint32_t *counter, void *stream) {
  return grpo_loss("aa_grpo_loss_seq", true, log_probs, lp_stride, ref_log_probs, ref_stride, old_log_probs, old_stride,
                   lp_dtype, advantages, completion_tokens, tok_stride, eos_id, B, K, beta, clip_low, clip_high,
                   dual_clip, loss_agg, kl_estimator, mode, loss, grad, grad_stride, clip_frac, row_end, scratch,
                   counter, stream, true);
}

extern "C" int aa_grpo_loss_topent(const void *log_probs, int64_t lp_stride, const void *ref_log_probs,
                                   int64_t ref_stride, const void *old_log_probs, int64_t old_stride, int lp_dtype,
                                   const float *advantages, const int64_t *completion_tokens, int64_t tok_stride,
                                   int64_t eos_id, int32_t B, int32_t K, float beta, float clip_low, float clip_high,
                                   float dual_clip, int loss_agg, int kl_estimator, int sequence, int mode, float *loss,
                                   void *grad, int64_t grad_stride, float *clip_frac, const float *entropy,
                                   int64_t ent_stride, const float *thr, int32_t *row_end, float *scratch,
                                   uint32_t *counter, void *stream) {
  AA_REQUIRE(sequence == 0 || sequence == 1, AA_ERR_ARG, "aa_grpo_loss_topent: sequence must be 0 or 1, got %d",
             sequence);
  return grpo_loss("aa_grpo_loss_topent", true, log_probs, lp_stride, ref_log_probs, ref_stride, old_log_probs,
                   old_stride, lp_dtype, advantages, completion_tokens, tok_stride, eos_id, B, K, beta, clip_low,
                   clip_high, dual_clip, loss_agg, kl_estimator, mode, loss, grad, grad_stride, clip_frac, row_end,
                   scratch, counter, stream, sequence == 1, true, entropy, ent_stride, thr);
}

extern "C" int aa_grpo_row_end(const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B,
                               int32_t K, int32_t *row_end, float *total, uint32_t *counter, void *stream) {
  AA_REQUIRE(B > 0 && K > 0 && completion_tokens && row_end && total && counter, AA_ERR_ARG,
             "aa_grpo_row_end: bad arguments");
  grpo_mask_kernel<128><<<B, 128, 0, static_cast<cudaStream_t>(stream)>>>(completion_tokens, tok_stride, B, K, eos_id,
                                                                          row_end, total, counter);
  return check_launch("aa_grpo_row_end");
}

// the checks both histogram passes share: exactly one of row_end / mask, sizes and strides
static int entropy_hist_args(const char *who, const float *entropy, int64_t ent_stride, const int32_t *row_end,
                             const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t K, const uint32_t *hist) {
  AA_REQUIRE(entropy && hist, AA_ERR_ARG, "%s: null pointer", who);
  AA_REQUIRE((row_end != nullptr) != (mask != nullptr), AA_ERR_ARG, "%s: give exactly one of row_end and mask", who);
  AA_REQUIRE(B > 0 && K > 0 && static_cast<int64_t>(B) * K <= INT32_MAX, AA_ERR_ARG, "%s: bad sizes (B=%d K=%d)", who,
             B, K);
  AA_REQUIRE(ent_stride >= K && (!mask || mask_stride >= K), AA_ERR_ARG, "%s: row strides must be >= K", who);
  return AA_OK;
}

static unsigned entropy_hist_grid(int32_t B, int32_t K) {
  const int64_t blocks = (static_cast<int64_t>(B) * K + 255) / 256;
  return static_cast<unsigned>(blocks < 1024 ? blocks : 1024);
}

extern "C" int aa_entropy_hist_hi(const float *entropy, int64_t ent_stride, const int32_t *row_end,
                                  const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t K, uint32_t *hist,
                                  void *stream) {
  int rc = entropy_hist_args("aa_entropy_hist_hi", entropy, ent_stride, row_end, mask, mask_stride, B, K, hist);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaMemsetAsync(hist, 0, sizeof(uint32_t) * (kEntBins + 1), st);
  entropy_hist_kernel<false><<<entropy_hist_grid(B, K), 256, 0, st>>>(entropy, ent_stride, row_end, mask, mask_stride,
                                                                      B, K, nullptr, hist);
  return check_launch("aa_entropy_hist_hi");
}

extern "C" int aa_entropy_select_hi(const uint32_t *hist, float q, uint32_t *sel, void *stream) {
  AA_REQUIRE(hist && sel, AA_ERR_ARG, "aa_entropy_select_hi: null pointer");
  AA_REQUIRE(q >= 0.f && q <= 1.f, AA_ERR_ARG, "aa_entropy_select_hi: q must lie in [0, 1], got %g", q);
  entropy_select_hi_kernel<<<1, kEntSelectThreads, 0, static_cast<cudaStream_t>(stream)>>>(hist, q, sel);
  return check_launch("aa_entropy_select_hi");
}

extern "C" int aa_entropy_hist_lo(const float *entropy, int64_t ent_stride, const int32_t *row_end,
                                  const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t K, const uint32_t *sel,
                                  uint32_t *hist, void *stream) {
  int rc = entropy_hist_args("aa_entropy_hist_lo", entropy, ent_stride, row_end, mask, mask_stride, B, K, hist);
  if (rc) return rc;
  AA_REQUIRE(sel, AA_ERR_ARG, "aa_entropy_hist_lo: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaMemsetAsync(hist, 0, sizeof(uint32_t) * 2 * kEntBins, st);
  entropy_hist_kernel<true><<<entropy_hist_grid(B, K), 256, 0, st>>>(entropy, ent_stride, row_end, mask, mask_stride,
                                                                     B, K, sel, hist);
  return check_launch("aa_entropy_hist_lo");
}

extern "C" int aa_entropy_select_lo(const uint32_t *hist, const uint32_t *sel, float *thr, void *stream) {
  AA_REQUIRE(hist && sel && thr, AA_ERR_ARG, "aa_entropy_select_lo: null pointer");
  entropy_select_lo_kernel<<<1, kEntSelectThreads, 0, static_cast<cudaStream_t>(stream)>>>(hist, sel, thr);
  return check_launch("aa_entropy_select_lo");
}

// the checks aa_cov_moments and aa_cov_keys share: exactly one of mask / row_end, sizes, strides and dtypes (fp32
// per-row advantages with row_end)
static int cov_rows(const char *who, const void *log_probs, int64_t lp_stride, int lp_dtype, const void *advantages,
                    int64_t adv_stride, int adv_dtype, const uint8_t *mask, int64_t mask_stride,
                    const int32_t *row_end, int32_t B, int32_t W, CovRows *out) {
  AA_REQUIRE(log_probs && advantages, AA_ERR_ARG, "%s: null pointer", who);
  AA_REQUIRE((row_end != nullptr) != (mask != nullptr), AA_ERR_ARG, "%s: give exactly one of row_end and mask", who);
  AA_REQUIRE(B > 0 && W > 0 && static_cast<int64_t>(B) * W <= INT32_MAX, AA_ERR_ARG, "%s: bad sizes (B=%d W=%d)", who,
             B, W);
  AA_REQUIRE(lp_stride >= W && (!mask || (mask_stride >= W && adv_stride >= W)), AA_ERR_ARG,
             "%s: row strides must be >= W", who);
  AA_REQUIRE(dtype_ok(lp_dtype) && dtype_ok(adv_dtype) && (mask || adv_dtype == AA_F32), AA_ERR_DTYPE,
             "%s: bad dtype (per-row advantages are fp32)", who);
  *out = CovRows{log_probs, lp_stride, lp_dtype, advantages, adv_stride, adv_dtype, mask, mask_stride, row_end, B, W};
  return AA_OK;
}

static unsigned cov_grid(int64_t n) {
  const int64_t blocks = (n + kCovThreads - 1) / kCovThreads;
  return static_cast<unsigned>(blocks < 1024 ? blocks : 1024);
}

extern "C" int aa_cov_moments(const void *log_probs, int64_t lp_stride, int lp_dtype, const void *advantages,
                              int64_t adv_stride, int adv_dtype, const uint8_t *mask, int64_t mask_stride,
                              const int32_t *row_end, int32_t B, int32_t W, uint32_t *state, void *stream) {
  CovRows c;
  int rc = cov_rows("aa_cov_moments", log_probs, lp_stride, lp_dtype, advantages, adv_stride, adv_dtype, mask,
                    mask_stride, row_end, B, W, &c);
  if (rc) return rc;
  AA_REQUIRE(state, AA_ERR_ARG, "aa_cov_moments: null state");
  cov_moments_kernel<<<1, kWhitenThreads, 0, static_cast<cudaStream_t>(stream)>>>(c, state);
  return check_launch("aa_cov_moments");
}

extern "C" int aa_cov_keys(int cov_mode, const void *log_probs, int64_t lp_stride, const void *old_log_probs,
                           int64_t old_stride, int lp_dtype, const void *advantages, int64_t adv_stride, int adv_dtype,
                           const uint8_t *mask, int64_t mask_stride, const int32_t *row_end, int32_t B, int32_t W,
                           float clip_low, float clip_high, float lb, float ub, uint32_t hash_seed, int mode,
                           const uint32_t *state, uint32_t *keys, uint8_t *elig, uint32_t *hist, void *stream) {
  CovRows c;
  int rc = cov_rows("aa_cov_keys", log_probs, lp_stride, lp_dtype, advantages, adv_stride, adv_dtype, mask,
                    mask_stride, row_end, B, W, &c);
  if (rc) return rc;
  AA_REQUIRE(state && keys && elig && hist, AA_ERR_ARG, "aa_cov_keys: null pointer");
  AA_REQUIRE(cov_mode == AA_COV_CLIP || cov_mode == AA_COV_KL, AA_ERR_ARG, "aa_cov_keys: unknown cov_mode %d",
             cov_mode);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "aa_cov_keys: bad mode");
  AA_REQUIRE(!old_log_probs || old_stride >= W, AA_ERR_ARG, "aa_cov_keys: old_stride must be >= W");
  AA_REQUIRE(cov_mode == AA_COV_KL || (actor_objective_ok(clip_low, clip_high, 0.f, AA_AGG_TOKEN_MEAN) && lb < ub &&
                                       isfinite(lb) && isfinite(ub)),
             AA_ERR_ARG, "aa_cov_keys: bad Clip-Cov arguments (need 0 <= clip_low < 1, clip_high >= 0, finite lb < ub; "
             "got %g %g %g %g)", clip_low, clip_high, lb, ub);
  const bool f = mode == AA_MODE_FAITHFUL;
  const CovKeyParams p{c, old_log_probs, old_stride, clip_low, clip_high, lb, ub, hash_seed,
                       f ? lp_dtype : AA_F32, f ? promote(lp_dtype, adv_dtype) : AA_F32, state, keys, elig, hist};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaMemsetAsync(hist, 0, sizeof(uint32_t) * kEntBins, st);
  const unsigned grid = cov_grid(static_cast<int64_t>(B) * W);
  if (cov_mode == AA_COV_KL)
    cov_keys_kernel<AA_COV_KL><<<grid, kCovThreads, 0, st>>>(p);
  else
    cov_keys_kernel<AA_COV_CLIP><<<grid, kCovThreads, 0, st>>>(p);
  return check_launch("aa_cov_keys");
}

extern "C" int aa_cov_select_hi(const uint32_t *hist, const double *ratio_host, uint32_t *state, void *stream) {
  AA_REQUIRE(hist && state && ratio_host, AA_ERR_ARG, "aa_cov_select_hi: null pointer");
  const double ratio = *ratio_host;
  AA_REQUIRE(ratio > 0.0 && ratio <= 1.0, AA_ERR_ARG, "aa_cov_select_hi: ratio must lie in (0, 1], got %g", ratio);
  cov_select_hi_kernel<<<1, kEntSelectThreads, 0, static_cast<cudaStream_t>(stream)>>>(hist, ratio, state);
  return check_launch("aa_cov_select_hi");
}

extern "C" int aa_cov_hist_lo(const uint32_t *keys, const uint8_t *elig, int64_t n, const uint32_t *state,
                              uint32_t *hist, void *stream) {
  AA_REQUIRE(keys && elig && state && hist, AA_ERR_ARG, "aa_cov_hist_lo: null pointer");
  AA_REQUIRE(n > 0 && n <= INT32_MAX, AA_ERR_ARG, "aa_cov_hist_lo: bad size %lld", static_cast<long long>(n));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaMemsetAsync(hist, 0, sizeof(uint32_t) * kEntBins, st);
  cov_hist_lo_kernel<<<cov_grid(n), kCovThreads, 0, st>>>(keys, elig, n, state, hist);
  return check_launch("aa_cov_hist_lo");
}

extern "C" int aa_cov_select_lo(const uint32_t *hist, uint32_t *state, float *share, void *stream) {
  AA_REQUIRE(hist && state && share, AA_ERR_ARG, "aa_cov_select_lo: null pointer");
  cov_select_lo_kernel<<<1, kEntSelectThreads, 0, static_cast<cudaStream_t>(stream)>>>(hist, state, share);
  return check_launch("aa_cov_select_lo");
}

extern "C" int aa_cov_mark(const uint32_t *keys, const uint8_t *elig, int32_t B, int32_t W, const uint32_t *state,
                           int32_t *tie_rows, uint8_t *sel, int64_t sel_stride, void *stream) {
  AA_REQUIRE(keys && elig && state && tie_rows && sel, AA_ERR_ARG, "aa_cov_mark: null pointer");
  AA_REQUIRE(B > 0 && W > 0 && static_cast<int64_t>(B) * W <= INT32_MAX && sel_stride >= W, AA_ERR_ARG,
             "aa_cov_mark: bad sizes (B=%d W=%d sel_stride=%lld)", B, W, static_cast<long long>(sel_stride));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cov_tie_kernel<<<B, kCovThreads, 0, st>>>(keys, elig, W, state, tie_rows);
  int rc = check_launch("aa_cov_mark(ties)");
  if (rc) return rc;
  cov_mark_kernel<<<B, kCovThreads, 0, st>>>(keys, elig, W, state, tie_rows, sel, sel_stride);
  return check_launch("aa_cov_mark");
}

extern "C" int aa_ppo_actor_loss_cov(const void *log_probs, int64_t lp_stride, const void *old_log_probs,
                                     int64_t old_stride, int lp_dtype, const void *advantages, int64_t adv_stride,
                                     int adv_dtype, const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t Wm,
                                     float clip_low, float clip_high, int loss_agg, int cov_mode, float cov_coef,
                                     const uint8_t *sel, int64_t sel_stride, int mode, const void *ref_log_probs,
                                     int64_t ref_stride, float kl_loss_coeff, int kl_estimator, float *loss,
                                     float *kl_loss, void *grad, int64_t grad_stride, float *clip_frac,
                                     float *row_scratch, uint32_t *counter, void *stream) {
  const char *who = "aa_ppo_actor_loss_cov";
  AA_REQUIRE(B > 0 && Wm > 0, AA_ERR_ARG, "%s: bad sizes", who);
  AA_REQUIRE(log_probs && old_log_probs && advantages && mask && sel && loss && row_scratch && counter, AA_ERR_ARG,
             "%s: null pointer", who);
  AA_REQUIRE(dtype_ok(lp_dtype) && dtype_ok(adv_dtype), AA_ERR_DTYPE, "%s: bad dtype", who);
  AA_REQUIRE(actor_objective_ok(clip_low, clip_high, 0.f, loss_agg), AA_ERR_ARG,
             "%s: bad objective (need 0 <= clip_low < 1, clip_high >= 0, a known loss_agg; got %g %g %d)", who,
             clip_low, clip_high, loss_agg);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "%s: bad mode", who);
  AA_REQUIRE(cov_mode == AA_COV_CLIP || cov_mode == AA_COV_KL, AA_ERR_ARG, "%s: unknown cov_mode %d", who, cov_mode);
  AA_REQUIRE(isfinite(cov_coef) && cov_coef >= 0.f, AA_ERR_ARG, "%s: cov_coef must be finite and >= 0, got %g", who,
             cov_coef);
  AA_REQUIRE(sel_stride >= Wm, AA_ERR_ARG, "%s: sel_stride must be >= Wm", who);
  if (ref_log_probs) {
    AA_REQUIRE(kl_estimator_ok(kl_estimator), AA_ERR_ARG, "%s: unknown kl_estimator code %d", who, kl_estimator);
    AA_REQUIRE(kl_loss_term_ok(kl_loss_coeff) && kl_loss, AA_ERR_ARG,
               "%s: a KL loss term needs kl_loss_coeff finite and > 0 (got %g) and kl_loss", who, kl_loss_coeff);
  }
  const bool f = (mode == AA_MODE_FAITHFUL);
  LossParams p{log_probs, lp_stride, old_log_probs, old_stride, lp_dtype, advantages, adv_stride, adv_dtype,
               mask, mask_stride, B, Wm, clip_low, f ? lp_dtype : AA_F32,
               f ? promote(lp_dtype, adv_dtype) : AA_F32, loss, grad, grad_stride, nullptr, row_scratch, counter, nullptr, 0,
               clip_high, 0.f, f ? adv_dtype : AA_F32, loss_agg, clip_frac, ref_log_probs, ref_stride,
               ref_log_probs ? kl_loss_coeff : 0.f, kl_estimator, kl_loss, sel, sel_stride, cov_coef};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (cov_mode == AA_COV_KL)
    ppo_loss_kernel<128, true, AA_COV_KL><<<B, 128, 0, st>>>(p);
  else
    ppo_loss_kernel<128, true, AA_COV_CLIP><<<B, 128, 0, st>>>(p);
  return check_launch(who);
}

extern "C" int aa_grpo_loss_cov(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                                const void *old_log_probs, int64_t old_stride, int lp_dtype, const float *advantages,
                                const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B,
                                int32_t K, float beta, float clip_low, float clip_high, int loss_agg, int kl_estimator,
                                int cov_mode, float cov_coef, const uint8_t *sel, int64_t sel_stride, int mode,
                                float *loss, void *grad, int64_t grad_stride, float *clip_frac, int32_t *row_end,
                                float *scratch, uint32_t *counter, void *stream) {
  AA_REQUIRE(cov_mode == AA_COV_CLIP || cov_mode == AA_COV_KL, AA_ERR_ARG, "aa_grpo_loss_cov: unknown cov_mode %d",
             cov_mode);
  AA_REQUIRE(isfinite(cov_coef) && cov_coef >= 0.f, AA_ERR_ARG,
             "aa_grpo_loss_cov: cov_coef must be finite and >= 0, got %g", cov_coef);
  AA_REQUIRE(sel && sel_stride >= K, AA_ERR_ARG, "aa_grpo_loss_cov: sel must be given with a row stride >= K");
  return grpo_loss("aa_grpo_loss_cov", true, log_probs, lp_stride, ref_log_probs, ref_stride, old_log_probs, old_stride,
                   lp_dtype, advantages, completion_tokens, tok_stride, eos_id, B, K, beta, clip_low, clip_high, 0.f,
                   loss_agg, kl_estimator, mode, loss, grad, grad_stride, clip_frac, row_end, scratch, counter, stream,
                   false, false, nullptr, 0, nullptr, cov_mode, cov_coef, sel, sel_stride);
}

extern "C" int aa_ppo_actor_loss_pm(const void *log_probs, int64_t lp_stride, const void *old_log_probs,
                                    int64_t old_stride, int lp_dtype, const void *advantages, int64_t adv_stride,
                                    int adv_dtype, const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t Wm,
                                    float clip_high, int loss_agg, int pm_mode, float tau_pos, float tau_neg, int mode,
                                    const void *ref_log_probs, int64_t ref_stride, float kl_loss_coeff,
                                    int kl_estimator, float *loss, float *kl_loss, void *grad, int64_t grad_stride,
                                    float *clip_frac, float *row_scratch, uint32_t *counter, void *stream) {
  const char *who = "aa_ppo_actor_loss_pm";
  AA_REQUIRE(B > 0 && Wm > 0, AA_ERR_ARG, "%s: bad sizes", who);
  AA_REQUIRE(log_probs && old_log_probs && advantages && mask && loss && row_scratch && counter, AA_ERR_ARG,
             "%s: null pointer", who);
  AA_REQUIRE(dtype_ok(lp_dtype) && dtype_ok(adv_dtype), AA_ERR_DTYPE, "%s: bad dtype", who);
  AA_REQUIRE(pm_mode_ok(pm_mode), AA_ERR_ARG, "%s: unknown pm_mode %d", who, pm_mode);
  AA_REQUIRE(actor_objective_ok(0.f, clip_high, 0.f, loss_agg), AA_ERR_ARG,
             "%s: bad objective (need clip_high >= 0 and a known loss_agg; got %g %d)", who, clip_high, loss_agg);
  AA_REQUIRE(sapo_temperature_ok(tau_pos) && sapo_temperature_ok(tau_neg), AA_ERR_ARG,
             "%s: tau_pos and tau_neg must be finite and > 0 (got %g %g)", who, tau_pos, tau_neg);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "%s: bad mode", who);
  if (ref_log_probs) {
    AA_REQUIRE(kl_estimator_ok(kl_estimator), AA_ERR_ARG, "%s: unknown kl_estimator code %d", who, kl_estimator);
    AA_REQUIRE(kl_loss_term_ok(kl_loss_coeff) && kl_loss, AA_ERR_ARG,
               "%s: a KL loss term needs kl_loss_coeff finite and > 0 (got %g) and kl_loss", who, kl_loss_coeff);
  }
  const bool f = (mode == AA_MODE_FAITHFUL);
  // s's dtype: the promoted one under CISPO, fp32 under SAPO (its temperature tensor is fp32)
  const int rp = (f && pm_mode == AA_PM_CISPO) ? promote(lp_dtype, adv_dtype) : AA_F32;
  LossParams p{log_probs, lp_stride, old_log_probs, old_stride, lp_dtype, advantages, adv_stride, adv_dtype,
               mask, mask_stride, B, Wm, 0.f, f ? lp_dtype : AA_F32, rp, loss, grad, grad_stride, nullptr, row_scratch,
               counter, nullptr, 0, clip_high, 0.f, f ? adv_dtype : AA_F32, loss_agg, clip_frac, ref_log_probs,
               ref_stride, ref_log_probs ? kl_loss_coeff : 0.f, kl_estimator, kl_loss, nullptr, 0, 0.f, tau_pos,
               tau_neg};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (pm_mode == AA_PM_SAPO)
    ppo_loss_kernel<128, true, AA_PM_SAPO><<<B, 128, 0, st>>>(p);
  else
    ppo_loss_kernel<128, true, AA_PM_CISPO><<<B, 128, 0, st>>>(p);
  return check_launch(who);
}

extern "C" int aa_grpo_loss_pm(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                               const void *old_log_probs, int64_t old_stride, int lp_dtype, const float *advantages,
                               const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B,
                               int32_t K, float beta, float clip_high, int loss_agg, int kl_estimator, int pm_mode,
                               float tau_pos, float tau_neg, int mode, float *loss, void *grad, int64_t grad_stride,
                               float *clip_frac, int32_t *row_end, float *scratch, uint32_t *counter, void *stream) {
  AA_REQUIRE(pm_mode_ok(pm_mode), AA_ERR_ARG, "aa_grpo_loss_pm: unknown pm_mode %d", pm_mode);
  AA_REQUIRE(sapo_temperature_ok(tau_pos) && sapo_temperature_ok(tau_neg), AA_ERR_ARG,
             "aa_grpo_loss_pm: tau_pos and tau_neg must be finite and > 0 (got %g %g)", tau_pos, tau_neg);
  return grpo_loss("aa_grpo_loss_pm", true, log_probs, lp_stride, ref_log_probs, ref_stride, old_log_probs, old_stride,
                   lp_dtype, advantages, completion_tokens, tok_stride, eos_id, B, K, beta, 0.f, clip_high, 0.f,
                   loss_agg, kl_estimator, mode, loss, grad, grad_stride, clip_frac, row_end, scratch, counter, stream,
                   false, false, nullptr, 0, nullptr, pm_mode, 0.f, nullptr, 0, tau_pos, tau_neg);
}

extern "C" int aa_nll_mean(const void *logp, int dtype, const int64_t *labels, int64_t n, int64_t ignore_index,
                           float *loss, float *neg_inv_count, float *partial, uint32_t *counter, void *stream) {
  AA_REQUIRE(n > 0 && logp && labels && loss && neg_inv_count && partial && counter, AA_ERR_ARG,
             "aa_nll_mean: bad arguments");
  AA_REQUIRE(dtype_ok(dtype), AA_ERR_DTYPE, "aa_nll_mean: bad dtype");
  int64_t blocks = (n + 255) / 256;
  if (blocks > 256) blocks = 256;
  nll_mean_kernel<256><<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      logp, dtype, labels, n, ignore_index, loss, neg_inv_count, partial, counter);
  return check_launch("aa_nll_mean");
}

static int make_coll(const aa_coll *coll, CollParams *out, const char *who) {
  *out = CollParams{nullptr, 0, 1, 0u, 0u};
  if (coll && coll->world > 1) {
    AA_REQUIRE(coll->peer_bufs && coll->world <= 32 && coll->rank >= 0 && coll->rank < coll->world, AA_ERR_ARG,
               "%s: bad collective descriptor", who);
    *out = CollParams{reinterpret_cast<float *const *>(coll->peer_bufs), coll->rank, coll->world, coll->epoch,
                      coll->max_lanes};
  }
  return AA_OK;
}

extern "C" int aa_ppo_pack_metrics(const float *row_stats, const float *reward, const float *value_row_mean,
                                   const float *actor_loss, const float *critic_loss, int32_t B, float *stats,
                                   const aa_coll *coll, const int32_t *status, void *stream) {
  AA_REQUIRE(B > 0 && row_stats && reward && stats, AA_ERR_ARG, "aa_ppo_pack_metrics: bad arguments");
  CollParams c;
  int rc = make_coll(coll, &c, "aa_ppo_pack_metrics");
  if (rc) return rc;
  ppo_pack_metrics_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(row_stats, reward, value_row_mean,
                                                                            actor_loss, critic_loss, B, stats, c, status);
  return check_launch("aa_ppo_pack_metrics");
}

extern "C" int aa_whiten_moments(const void *advantages, int adv_dtype, int64_t adv_row_stride, const uint8_t *mask,
                                 int64_t mask_row_stride, int32_t B, int32_t W, double *moments, int32_t k, int32_t K,
                                 void *stream) {
  AA_REQUIRE(advantages && mask && moments, AA_ERR_ARG, "aa_whiten_moments: null pointer");
  AA_REQUIRE(dtype_ok(adv_dtype), AA_ERR_DTYPE, "aa_whiten_moments: bad dtype %d", adv_dtype);
  AA_REQUIRE(B > 0 && W > 0 && static_cast<int64_t>(B) * W <= INT32_MAX, AA_ERR_ARG,
             "aa_whiten_moments: bad sizes (B=%d W=%d)", B, W);
  AA_REQUIRE(adv_row_stride >= W && mask_row_stride >= W, AA_ERR_ARG, "aa_whiten_moments: row strides must be >= W");
  AA_REQUIRE(K > 0 && k >= 0 && k < K, AA_ERR_ARG, "aa_whiten_moments: slot k=%d outside [0, K=%d)", k, K);
  whiten_moments_kernel<<<1, kWhitenThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      advantages, adv_dtype, adv_row_stride, mask, mask_row_stride, B, W, moments + 3 * static_cast<int64_t>(k));
  return check_launch("aa_whiten_moments");
}

extern "C" int aa_whiten_reduce(const double *moments, int32_t K, double *total, void *stream) {
  AA_REQUIRE(moments && total, AA_ERR_ARG, "aa_whiten_reduce: null pointer");
  AA_REQUIRE(K > 0, AA_ERR_ARG, "aa_whiten_reduce: bad slot count K=%d", K);
  whiten_reduce_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(moments, K, total);
  return check_launch("aa_whiten_reduce");
}

extern "C" int aa_whiten_apply(void *advantages, int adv_dtype, int64_t adv_row_stride, const uint8_t *mask,
                               int64_t mask_row_stride, int32_t B, int32_t W, const double *total, int32_t *status,
                               void *stream) {
  AA_REQUIRE(advantages && mask && total && status, AA_ERR_ARG, "aa_whiten_apply: null pointer");
  AA_REQUIRE(dtype_ok(adv_dtype), AA_ERR_DTYPE, "aa_whiten_apply: bad dtype %d", adv_dtype);
  AA_REQUIRE(B > 0 && W > 0 && B <= 65535, AA_ERR_ARG, "aa_whiten_apply: bad sizes (B=%d W=%d)", B, W);
  AA_REQUIRE(adv_row_stride >= W && mask_row_stride >= W, AA_ERR_ARG, "aa_whiten_apply: row strides must be >= W");
  const dim3 grid((W + 255) / 256, B);
  whiten_apply_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(advantages, adv_dtype, adv_row_stride, mask,
                                                                           mask_row_stride, W, total, status);
  return check_launch("aa_whiten_apply");
}

extern "C" int aa_allreduce_packed(const float *src, float *dst, int32_t n, const aa_coll *coll, void *stream) {
  AA_REQUIRE(src && dst && n > 0 && n <= kCollLanes && coll, AA_ERR_ARG, "aa_allreduce_packed: bad arguments (n <= 16)");
  CollParams c;
  int rc = make_coll(coll, &c, "aa_allreduce_packed");
  if (rc) return rc;
  if (c.world <= 1) {
    if (src != dst) cudaMemcpyAsync(dst, src, sizeof(float) * n, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream));
    return check_launch("aa_allreduce_packed");
  }
  allreduce_packed_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(src, dst, n, c);
  return check_launch("aa_allreduce_packed");
}
