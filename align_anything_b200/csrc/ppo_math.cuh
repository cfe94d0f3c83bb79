// ppo_math.cuh -- per-token arithmetic of the PPO actor loss with the reference's rounding points, shared by K5
// (ppo.cu: ppo_loss_kernel) and the single-pass actor node (logprob_fused.cu), so that both produce the same bits.
//
// trainers/text_to_text/ppo.py:291-307 (actor_loss_fn) + utils/tools.py:460-467 (masked_mean) and the autograd chain
// Mean -> Div -> Sum -> Mul(mask) -> Maximum -> Mul -> Clamp -> Exp -> Sub restated per token.
#pragma once

#include "common.cuh"

namespace aa {

// upstream coefficient of d loss / d (row sum of the masked objective): -(1/B)/cnt, rounded where the eager ops round
// (`rp` = promoted dtype of log-probs and advantages).  The count is the int64 `mask.sum(-1)`, which ATen casts to `rp`
// before it divides (a bf16 row of 257 tokens is divided by 256), in the forward and in DivBackward alike.
__device__ __forceinline__ float actor_row_coeff(float cnt, int B, int rp) {
  const float g_q = round_to(-1.f / static_cast<float>(B), rp);
  return round_to(g_q / round_to(cnt, rp), rp);
}

// upstream coefficient under token-mean aggregation, -(s * mask).sum() / mask.sum():  -1 / total (DivBackward's
// rounding), total = the micro-batch's masked-in token count, cast to `rp` by ATen CUDA like the row count above
__device__ __forceinline__ float actor_token_mean_coeff(float total, int rp) {
  return round_to(-1.f / round_to(total, rp), rp);
}

// d total / d KL of a masked-in token for the actor's KL loss term  kl_coeff * agg(KL, mask)  (K5 and K1f's
// aa_*_kl entry points).  The KL has the log-probs' dtype (rounding code r), and so has every op of its chain:
//   seq-mean-token-mean  round(round(round(c) * (1/B)) / round(count))   MulBackward by the python scalar c, then
//                        MeanBackward (ATen CUDA multiplies by the reciprocal of a scalar divisor), then DivBackward
//                        by the row's int64 mask count cast to r;  count = the row's masked-in tokens
//   token-mean           round(round(c) / round(count))                  count = the micro-batch's masked-in tokens
__device__ __forceinline__ float kl_term_coeff(float kl_coeff, int agg, float count, int B, int r) {
  const float g = round_to(kl_coeff, r);
  if (agg == AA_AGG_TOKEN_MEAN) return round_to(g / round_to(count, r), r);
  return round_to(round_to(g * (1.f / static_cast<float>(B)), r) / round_to(count, r), r);
}

// the argument check of the KL loss term of the actor entry points (the trainers check the same on the host)
inline bool kl_loss_term_ok(float kl_coeff) { return kl_coeff > 0.f && kl_coeff <= 3.402823466e38f; }

// the argument check of the objective entry points (ops.ActorObjective checks the same on the host)
inline bool actor_objective_ok(float clip_low, float clip_high, float dual_clip, int loss_agg) {
  return clip_low >= 0.f && clip_low < 1.f && clip_high >= 0.f && (dual_clip == 0.f || dual_clip > 1.f) &&
         (loss_agg == AA_AGG_SEQ_MEAN_TOKEN_MEAN || loss_agg == AA_AGG_TOKEN_MEAN);
}

// The clip / tie / dual-clip arithmetic of actor_token at a given ratio (rounding code rx) and clip bounds lo / hi
// (already rounded to rx), shared by the token-level ratio (actor_token below) and GRPO's sequence-level
// ratio (grpo_seq_row).  gs: the gradient reaching `ratio` (0 when `on` is false); obj, why: as actor_token's.
__device__ __forceinline__ void clipped_ratio(float ratio, float lo, float hi, float aux, bool on, float g_rs,
                                              float dual, int rx, int rp, int ra, float &obj, float &gs, int &why) {
  const float s1 = round_to(aux * ratio, rp);
  const float clipped = fminf(fmaxf(ratio, lo), hi);
  const float s2 = round_to(aux * clipped, rp);
  obj = fminf(s1, s2);
  if (s1 != s1 || s2 != s2) obj = NAN;
  why = (s2 < s1) ? 1 : 0;
  float g = g_rs;  // gradient reaching min(s1, s2)
  if (dual != 0.f && aux < 0.f) {
    // maximum's backward: all to the larger input, round(grad / 2) to each on a tie; the c * adv branch does not
    // reach the ratio
    const float ca = round_to(dual * aux, ra);
    if (obj < ca) {
      g = 0.f;
      why |= 2;
    } else if (obj == ca) {
      g = round_to(0.5f * g_rs, rp);
    }
    if (obj == obj) obj = fmaxf(obj, ca);
  }
  const bool in_range = (ratio >= lo) && (ratio <= hi);
  gs = 0.f;  // gradient reaching `ratio` through both branches of torch.minimum
  if (on) {
    if (s1 < s2) {
      gs = round_to(round_to(g * aux, rp), rx);
    } else if (s1 == s2) {
      // a tie: minimum's backward sends round(grad / 2) down each branch; through the clamp only in range, and the
      // ratio's gradient is the sum of the two (rounded at each step: the halves differ from g * aux / 2 once they
      // are fp16 subnormals)
      const float half = round_to(round_to(round_to(0.5f * g, rp) * aux, rp), rx);
      gs = in_range ? round_to(half + half, rx) : half;
    }
    // s1 > s2: the clipped branch wins and clamp's backward is zero outside the range
  }
}

// One token of the clipped-ratio objective.  x / old: new / old log-prob (dtype code rx), aux: advantage,
// on: the mask bit, g_rs: d loss / d (the token's objective) for a masked-in token (actor_row_coeff or
// actor_token_mean_coeff).  eps_lo / eps_hi: the clip range [1 - eps_lo, 1 + eps_hi]; dual: the dual-clip factor c
// (0 = off), ra: the rounding code of `c * adv` (the advantages' dtype).
//   obj  = min(adv * ratio, adv * clip(ratio))     (the NEGATED loss term; NaN-propagating like torch.minimum)
//          dual-clip, adv < 0:  max(obj, c * adv)  (torch.where(adv < 0, torch.maximum(obj, c * adv), obj))
//   grad = d loss / d x                            (0 when the mask is off)
//   why  = bit 0: the clipped branch is strictly smaller; bit 1: c * adv wins (the clip-fraction counters)
__device__ __forceinline__ void actor_token(float x, float old, float aux, bool on, float g_rs, float eps_lo,
                                            float eps_hi, float dual, int rx, int rp, int ra, float &obj, float &grad,
                                            int &why) {
  const float lo = round_to(1.f - eps_lo, rx), hi = round_to(1.f + eps_hi, rx);
  const float ratio = round_to(expf(round_to(x - old, rx)), rx);
  float gs;
  clipped_ratio(ratio, lo, hi, aux, on, g_rs, dual, rx, rp, ra, obj, gs, why);
  grad = round_to(gs * ratio, rx);  // ExpBackward: grad * result
}

// One token of Clip-Cov / KL-Cov (verl's compute_policy_loss_clip_cov / _kl_cov; tests/cov_port.py is the
// specification), `sel` the token's bit of the covariance selection:
//   AA_COV_CLIP  actor_token's clip-higher objective (no dual-clip); a selected token's objective and gradient are 0
//   AA_COV_KL    the unclipped s = adv * ratio; a selected token takes s - kl_coef * |x - old|, whose gradient
//                through |.| is sign(x - old) (0 at 0)
// x, old, aux, on, g_rs, rx, rp, obj, grad, why: as actor_token's (KL-Cov clips nothing: why = 0).
__device__ __forceinline__ void cov_token(int mode, float x, float old, float aux, bool on, bool sel, float g_rs,
                                          float eps_lo, float eps_hi, float kl_coef, int rx, int rp, float &obj,
                                          float &grad, int &why) {
  if (mode == AA_COV_CLIP) {
    actor_token(x, old, aux, on, g_rs, eps_lo, eps_hi, 0.f, rx, rp, rp, obj, grad, why);
    if (sel) obj = grad = 0.f;
    return;
  }
  const float d = round_to(x - old, rx);
  const float ratio = round_to(expf(d), rx);
  obj = round_to(aux * ratio, rp);
  why = 0;
  grad = 0.f;
  if (sel) obj = round_to(obj - round_to(kl_coef * fabsf(d), rx), rp);
  if (!on) return;
  grad = round_to(round_to(round_to(g_rs * aux, rp), rx) * ratio, rx);  // through the ratio (ExpBackward)
  if (sel && d != 0.f) {  // through -kl_coef * |d|: MulBackward by the scalar, then AbsBackward's sign.  kl_coef * |d|
    // has the log-probs' dtype, so the gradient reaching it is rounded to rx first (a no-op unless rp is wider, as
    // with GRPO's or PPO's fp32 advantages under 16-bit log-probs)
    const float ga = round_to(round_to(-g_rs, rx) * kl_coef, rx);
    grad = round_to(grad + (d > 0.f ? ga : -ga), rx);
  }
}

// ---- CISPO and SAPO (ops.POLICY_LOSS_MODES 'cispo' / 'sapo'; tests/policy_loss_port.py is the specification) ----
// the argument checks of the AA_PM_* entry points (ops.ActorObjective checks the same on the host)
inline bool pm_mode_ok(int pm) { return pm == AA_PM_CISPO || pm == AA_PM_SAPO; }
inline bool sapo_temperature_ok(float tau) { return tau > 0.f && tau <= 3.402823466e38f; }

// One token of CISPO (MiniMax-M1) or SAPO (Qwen's Soft Adaptive Policy Optimization).  x, old, aux, on, g_rs, rx, obj,
// grad: as actor_token's; rp: the dtype of s (the promoted dtype under CISPO; fp32 under SAPO, whose temperature
// tensor is fp32).  ratio = exp(x - old) in rx.
//   AA_PM_CISPO  w = clamp(ratio, max = round_rx(1 + eps_hi)), detached (NaN stays NaN);  obj = s = (w * aux) * x
//                grad = round_rx(round_rp(g_rs * (w * aux)))      (MulBackward; nothing reaches the ratio)
//                why bit 0: ratio > the bound (the clip-fraction counter)
//   AA_PM_SAPO   tau = aux > 0 ? tau_pos : tau_neg;  sig = 1 / (1 + exp(-(tau * (ratio - 1))));  obj = ((sig * 4) / tau) * aux
//                the backward op for op: Mul by aux, Div by tau, Mul by 4, SigmoidBackward ((g * (1 - sig)) * sig), Mul by
//                tau (cast to rx), ExpBackward (* ratio);  why = 0
__device__ __forceinline__ void pm_token(int pm, float x, float old, float aux, bool on, float g_rs, float eps_hi,
                                         float tau_pos, float tau_neg, int rx, int rp, float &obj, float &grad,
                                         int &why) {
  const float ratio = round_to(expf(round_to(x - old, rx)), rx);
  grad = 0.f;
  why = 0;
  if (pm == AA_PM_CISPO) {
    const float hi = round_to(1.f + eps_hi, rx);
    const bool over = ratio > hi;
    const float wa = round_to((over ? hi : ratio) * aux, rp);
    obj = round_to(wa * x, rp);
    why = over ? 1 : 0;
    if (on) grad = round_to(round_to(g_rs * wa, rp), rx);
    return;
  }
  const float tau = aux > 0.f ? tau_pos : tau_neg;
  const float sig = 1.f / (1.f + expf(-(tau * round_to(ratio - 1.f, rx))));
  obj = ((sig * 4.f) / tau) * aux;
  if (on) {
    const float gu = ((((g_rs * aux) / tau) * 4.f) * (1.f - sig)) * sig;
    grad = round_to(round_to(gu * tau, rx) * ratio, rx);
  }
}

// ---- KL estimators (ops.KL_ESTIMATORS; tests/kl_objective_port.py is their specification) ---------------------
// One token's estimate of KL(policy || reference) from the log-probs lp and rf, each op rounded to `r` as the eager
// expression rounds it:
//   AA_KL_K1  lp - rf
//   AA_KL_K2  0.5 * (lp - rf) ** 2
//   AA_KL_K3  exp(rf - lp) - (rf - lp) - 1      (the reference GRPO's expression, op for op)
// aux: what kl_grad needs of the forward (k2: lp - rf; k3: exp(rf - lp)).
inline bool kl_estimator_ok(int est) { return est == AA_KL_K1 || est == AA_KL_K2 || est == AA_KL_K3; }

__device__ __forceinline__ float kl_value(float lp, float rf, int est, int r, float &aux) {
  if (est == AA_KL_K3) {
    const float d = round_to(rf - lp, r);
    aux = round_to(expf(d), r);
    return round_to(round_to(aux - d, r) - 1.f, r);
  }
  const float d = round_to(lp - rf, r);
  aux = d;
  if (est == AA_KL_K1) return d;
  return round_to(0.5f * round_to(d * d, r), r);  // pow(d, 2) is d * d on ATen CUDA
}

// d loss / d lp of a token: `acc` (the gradient that reaches lp through the other terms, accumulated first: autograd
// runs the later-created ratio node before the KL's) plus what g_kl = d loss / d KL sends through the estimator:
//   k1  acc + g_kl
//   k2  acc + round(round(0.5 * g_kl) * (2 * d))                    (MulBackward, then PowBackward's grad * (2 * d))
//   k3  (acc + g_kl) - round(g_kl * e)                              (the linear term first, then ExpBackward)
__device__ __forceinline__ float kl_grad(float acc, float g_kl, int est, float aux, int r) {
  if (est == AA_KL_K3) return round_to(round_to(acc + g_kl, r) - round_to(g_kl * aux, r), r);
  if (est == AA_KL_K1) return round_to(acc + g_kl, r);
  return round_to(acc + round_to(round_to(0.5f * g_kl, r) * (2.f * aux), r), r);
}

// ---- GRPO (trainers/text_to_text/grpo.py:290-312) ---------------------------------------------------------
// One token of  -(exp(lp - lp.detach()) * A - beta * KL),  KL = exp(ref - lp) - (ref - lp) - 1 (k3 estimator), with the
// reference's rounding points when lp is 16-bit (`r`).  g_t = 1 / (number of counted tokens): d loss / d per-token loss.
//   ptl  = the per-token loss (exp(lp - lp.detach()) == 1 exactly)
//   grad = d loss / d lp; three contributions reach lp and are accumulated in the order autograd's engine runs the nodes
//          (later-created first):  c1 = round(-g_t * A)  through exp(lp - lp.detach()) * A;
//          c3 = +g_kl  through the linear term -(ref - lp) of the KL, g_kl = round(round(g_t) * beta);
//          c2 = -round(g_kl * e)  through exp(ref - lp)
__device__ __forceinline__ void grpo_token(float lp, float rf, float A, bool on, float g_t, float beta, int r, float &ptl,
                                           float &grad) {
  const float d = round_to(rf - lp, r);
  const float e = round_to(expf(d), r);
  const float kl = round_to(round_to(e - d, r) - 1.f, r);
  const float bk = round_to(beta * kl, r);
  ptl = -(A - bk);
  grad = 0.f;
  if (on) {
    const float c1 = round_to(-g_t * A, r);
    const float g_kl = round_to(round_to(g_t, r) * beta, r);
    const float c2 = -round_to(g_kl * e, r);
    grad = round_to(round_to(c1 + g_kl, r) + c2, r);
  }
}

// the argument check of the GRPO objective entry points: the actor objective's ranges, and GRPO's third aggregation
// (ops.GrpoObjective checks the same on the host)
inline bool grpo_objective_ok(float clip_low, float clip_high, float dual_clip, int loss_agg) {
  return actor_objective_ok(clip_low, clip_high, dual_clip, AA_AGG_TOKEN_MEAN) &&
         (loss_agg == AA_AGG_TOKEN_MEAN || loss_agg == AA_AGG_SEQ_MEAN_TOKEN_MEAN ||
          loss_agg == AA_AGG_SEQ_MEAN_TOKEN_SUM_NORM);
}

// d loss / d per-token loss of a counted token under each GRPO aggregation, as the eager ops round it (fp32: the
// per-token loss is fp32 because the advantages are):  token-mean  1 / total ;  seq-mean-token-mean  (1 / B) / cnt_b
// (MeanBackward, then DivBackward by the row's count) ;  seq-mean-token-sum-norm  1 / (B * K)
__device__ __forceinline__ float grpo_agg_coeff(int agg, float total, float cnt, int B, int K) {
  if (agg == AA_AGG_SEQ_MEAN_TOKEN_MEAN) return (1.f / static_cast<float>(B)) / cnt;
  if (agg == AA_AGG_SEQ_MEAN_TOKEN_SUM_NORM) return 1.f / (static_cast<float>(B) * static_cast<float>(K));
  return 1.f / total;
}

// One token of GRPO's clipped objective (DeepSeekMath's GRPO with clip-higher and dual-clip):
//   -(s - beta * KL),  s = the clipped-ratio objective of actor_token with r = exp(lp - old), old = the rollout-time
// policy log-prob, and the k3 KL of grpo_token.  g_t: d loss / d per-token loss (grpo_agg_coeff).  The advantage is
// fp32, so s and the per-token loss are fp32 (actor_token's promoted and `c * A` roundings are fp32); `r` rounds what
// has the log-prob dtype.  The gradient reaching lp through the ratio takes c1's place in grpo_token's accumulation
// order (the ratio is created after the KL, as the reference creates its exp(lp - lp.detach()) term).  est: the KL
// estimator (AA_KL_K3 is the reference's; kl_value / kl_grad).
//   why: actor_token's clip-fraction bits
// keep: the top-entropy mask (aa_grpo_loss_topent), 1 or 0: the per-token loss is -(s * keep - beta * KL), so a
// masked token (keep 0) carries the KL term alone and s sends it no gradient; the clip-fraction bits stay the token's
__device__ __forceinline__ void grpo_obj_token(float lp, float old, float rf, float A, bool on, float g_t, float beta,
                                               float eps_lo, float eps_hi, float dual, int est, int r, float &ptl,
                                               float &grad, int &why, float keep = 1.f) {
  float s, ga, aux;
  actor_token(lp, old, A, on, -g_t * keep, eps_lo, eps_hi, dual, r, AA_F32, AA_F32, s, ga, why);
  const float kl = kl_value(lp, rf, est, r, aux);
  const float bk = round_to(beta * kl, r);
  ptl = -(s * keep - bk);
  grad = 0.f;
  if (on) grad = kl_grad(ga, round_to(round_to(g_t, r) * beta, r), est, aux, r);
}

// One token of GRPO under Clip-Cov / KL-Cov (aa_grpo_loss_cov): -(s - beta * KL) with cov_token's s (fp32, as
// grpo_obj_token's) and grpo_obj_token's KL and accumulation order
__device__ __forceinline__ void grpo_cov_token(int mode, float lp, float old, float rf, float A, bool on, bool sel,
                                               float g_t, float beta, float eps_lo, float eps_hi, float kl_coef,
                                               int est, int r, float &ptl, float &grad, int &why) {
  float s, ga, aux;
  cov_token(mode, lp, old, A, on, sel, -g_t, eps_lo, eps_hi, kl_coef, r, AA_F32, s, ga, why);
  const float kl = kl_value(lp, rf, est, r, aux);
  ptl = -(s - round_to(beta * kl, r));
  grad = 0.f;
  if (on) grad = kl_grad(ga, round_to(round_to(g_t, r) * beta, r), est, aux, r);
}

// One token of GRPO under CISPO / SAPO (aa_grpo_loss_pm, K1f's kind 3 with the mode): -(s - beta * KL) with
// pm_token's s (fp32: the advantage is fp32) and grpo_obj_token's KL and accumulation order
__device__ __forceinline__ void grpo_pm_token(int pm, float lp, float old, float rf, float A, bool on, float g_t,
                                              float beta, float eps_hi, float tau_pos, float tau_neg, int est, int r,
                                              float &ptl, float &grad, int &why) {
  float s, ga, aux;
  pm_token(pm, lp, old, A, on, -g_t, eps_hi, tau_pos, tau_neg, r, AA_F32, s, ga, why);
  const float kl = kl_value(lp, rf, est, r, aux);
  ptl = -(s - round_to(beta * kl, r));
  grad = 0.f;
  if (on) grad = kl_grad(ga, round_to(round_to(g_t, r) * beta, r), est, aux, r);
}

// GSPO's sequence-level ratio for one row (aa_grpo_loss_seq; tests/gspo_port.py is the specification):
//   S = round_r(sum_t (lp_t - old_t) * m_t)   the row's summed log-ratio, in the log-prob dtype (`r`)
//   log_w = S / n,  w = exp(log_w)           fp32 (n = the row's fp32 token count), and so are the clip bounds
//   s = clipped_ratio(w) with fp32 roundings  the row's objective, shared by its tokens
// g_t: d loss / d per-token loss of a counted token (grpo_agg_coeff), so d loss / d s = -n * g_t, the sum of the
// row's per-token coefficients.  coef = d loss / d lp_t through the ratio, the same for every masked-in token:
// ExpBackward (gs * w), DivBackward by n, cast once to `r` at the backward of the sum.  why: clipped_ratio's bits.
// n_s: the counted tokens whose per-token loss takes s -- n, or under the top-entropy mask the row's kept tokens, so
// d loss / d s = -n_s * g_t while the ratio's gradient still reaches every counted token through the row's mean.
__device__ __forceinline__ void grpo_seq_row(float S, float n, float n_s, float A, float g_t, float eps_lo,
                                             float eps_hi, float dual, int r, float &s, float &coef, int &why) {
  const float w = expf(S / n);
  float gs;
  clipped_ratio(w, 1.f - eps_lo, 1.f + eps_hi, A, true, -(n_s * g_t), dual, AA_F32, AA_F32, AA_F32, s, gs, why);
  coef = round_to((gs * w) / n, r);
}

// One token of GSPO's loss: -(s - beta * KL) with the row's objective s and ratio coefficient coef (grpo_seq_row),
// and grpo_obj_token's KL and accumulation order (the ratio's gradient first, then the KL's)
__device__ __forceinline__ void grpo_seq_token(float lp, float rf, float s, float coef, bool on, float g_t, float beta,
                                               int est, int r, float &ptl, float &grad) {
  float aux;
  const float kl = kl_value(lp, rf, est, r, aux);
  const float bk = round_to(beta * kl, r);
  ptl = -(s - bk);
  grad = 0.f;
  if (on) grad = kl_grad(coef, round_to(round_to(g_t, r) * beta, r), est, aux, r);
}

// pass 1: first eos per row (-> row_end[b] = number of counted tokens) and the global token count
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
    grpo_mask_kernel(const int64_t *__restrict__ tokens, int64_t tok_stride, int B, int K, int64_t eos_id,
                     int32_t *__restrict__ row_end, float *__restrict__ total, uint32_t *counter) {
  __shared__ int sh_min;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) sh_min = K;
  __syncthreads();
  int first = K;
  for (int t = threadIdx.x; t < K; t += THREADS)
    if (tokens[b * tok_stride + t] == eos_id) first = min(first, t);
  if (first < K) atomicMin(&sh_min, first);
  __syncthreads();
  if (threadIdx.x == 0) row_end[b] = (sh_min < K) ? sh_min + 1 : K;  // mask[t] = 1 for t <= first eos
  if (!last_block_arrives(counter, gridDim.x)) return;
  if (threadIdx.x == 0) {
    const volatile int32_t *re = row_end;
    float c = 0.f;
    for (int i = 0; i < B; ++i) c += static_cast<float>(re[i]);
    total[0] = c;
  }
}


}  // namespace aa
