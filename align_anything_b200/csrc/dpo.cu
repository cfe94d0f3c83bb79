// dpo.cu -- K2: DPO pairwise log-sigmoid loss + metrics + the per-sample upstream gradient
// for K1b, and the pad-stripping label extraction that precedes K1 in the DPO trainers.
//
// Replaces trainers/text_to_text/dpo.py:52-54,135-137 (strip_pad tail), :166-203 (loss loop:
// ~12 tiny kernels per pair in the reference) and :215-221 (local metric means);
// trainers/text_audio_to_text/dpo.py:134-139 (identical pairs are dropped).
#include "common.cuh"

namespace aa {

// ---- labels = strip_pad(input_ids[i])[-R_i:] --------------------------------------------------
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
    strip_pad_tail_kernel(const int64_t *__restrict__ ids, int L, int64_t row_stride, int64_t pad,
                          int strip, const int32_t *__restrict__ lens, int64_t *__restrict__ out,
                          int64_t out_stride, int32_t *status) {
  constexpr int NW = THREADS / kWarp;
  __shared__ int warp_cnt[NW];
  const int i = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int R = lens[i];
  const int64_t *row = ids + static_cast<int64_t>(i) * row_stride;
  int64_t *dst = out + static_cast<int64_t>(i) * out_stride;
  if (R <= 0) return;
  if (!strip) {
    if (R > L) {
      if (tid == 0 && status) atomicOr(status, AA_STATUS_SHORT_SEQUENCE);
      for (int k = tid; k < R; k += THREADS) dst[k] = (k >= R - L) ? row[L - R + k] : -1;
      return;
    }
    for (int k = tid; k < R; k += THREADS) dst[k] = row[L - R + k];
    return;
  }
  int carry = 0;  // non-pad tokens seen so far, scanning right to left
  for (int base = L - 1; base >= 0 && carry < R; base -= THREADS) {
    const int pos = base - tid;
    int64_t v = 0;
    bool keep = false;
    if (pos >= 0) {
      v = row[pos];
      keep = (v != pad);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    const int in_warp = __popc(bal & ((2u << lane) - 1u));  // inclusive rank inside the warp
    if (lane == 31) warp_cnt[wid] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < NW; ++w) {
      const int c = warp_cnt[w];
      before += (w < wid) ? c : 0;
      total += c;
    }
    const int rank = carry + before + in_warp;  // 1-based rank from the right among non-pads
    if (keep && rank <= R) dst[R - rank] = v;
    carry += total;
    __syncthreads();
  }
  if (carry < R) {  // fewer non-pad tokens than response_len: the reference would mis-shape
    if (tid == 0 && status) atomicOr(status, AA_STATUS_SHORT_SEQUENCE);
    for (int k = tid; k < R - carry; k += THREADS) dst[k] = -1;
  }
}

// ---- K2 -------------------------------------------------------------------------------------
struct DpoParams {
  const void *policy_lp;
  const void *ref_lp;
  int lp_dtype;
  int n_pairs;
  int width;
  int64_t row_stride;
  float beta;
  int round_dt;  // dtype whose rounding the reference applies at each op (AA_F32: none)
  const int64_t *ids;
  int L;
  int64_t ids_row_stride;
  float *per_pair;
  float *grad_seg;
  float *stats;
  uint32_t *counter;
  float *stats_global;  // optional: the all-reduced stats (fused collective), else unused
  CollParams coll;      // coll.world <= 1: no collective
  const int32_t *status;  // optional: device status word, copied into stats[7] (MAX lane of the step's all-reduce)
};

// K2 with the objective options (DESIGN section 4.5).  A type of its own, so that the reference loss's
// instantiation keeps its parameter block, and its code, as they were.
struct DpoObjParams : DpoParams {
  int loss_type;          // AA_DPO_*
  float eps;              // label_smoothing
  float alpha;            // rpo_alpha: 0 = no NLL term
  const int32_t *counts;  // optional: scored rows per sample (R_i - 1), [2 * n_pairs]
};

template <int THREADS>
__device__ __forceinline__ float row_sum(const void *base, int dt, int64_t off, int width, float *scratch) {
  float acc = 0.f;
  for (int k = threadIdx.x; k < width; k += THREADS) acc += load_as_float(base, off + k, dt);
  return block_sum<THREADS>(acc, scratch);
}

__device__ __forceinline__ float log_sigmoid(float z) {
  // ATen log_sigmoid forward: min(z, 0) - log1p(exp(-|z|))
  return fminf(z, 0.f) - log1pf(expf(-fabsf(z)));
}
__device__ __forceinline__ float dlog_sigmoid(float z) {
  // ATen log_sigmoid_backward: max_deriv - sign * (e / (1 + e)), e = exp(-|z|)
  const float e = expf(-fabsf(z));
  const bool neg = z < 0.f;
  return (neg ? 1.f : 0.f) - (neg ? 1.f : -1.f) * (e / (1.f + e));
}

// ---- K2 objective options (DESIGN section 4.5) ----------------------------------------------
// Each loss restates tests/dpo_objective_port.py op for op: FAITHFUL rounds (rd) wherever the port's eager op on a
// 0-dim tensor of the log-prob dtype rounds, and every product is __fmul_rn so that no rounding point is contracted
// away.  The forward keeps two floats per pair (s0, s1) from which the last block, once it knows 1 / n_kept, runs the
// port's autograd chain.  a = pc - rc, b = pr - rr (IPO: each sum divided by its row count first).
struct DpoPairFwd {
  float loss, s0, s1;
};

__device__ __forceinline__ float sigmoid_f(float z) { return 1.f / (1.f + expf(-z)); }

__device__ __forceinline__ DpoPairFwd dpo_obj_forward(int type, float a, float b, float beta, float eps, int rd) {
  const float c = static_cast<float>(0.5 / static_cast<double>(beta));  // 1 / (2 beta)
  DpoPairFwd f{0.f, 0.f, 0.f};
  switch (type) {
    case AA_DPO_SIGMOID:
    case AA_DPO_ROBUST: {
      const float z = round_to(__fmul_rn(beta, round_to(a - b, rd)), rd);
      const float t1 = round_to(log_sigmoid(z), rd);
      f.loss = -t1;
      if (eps != 0.f) {
        const float m1 = round_to(__fmul_rn(-t1, 1.f - eps), rd);
        const float m2 = round_to(__fmul_rn(round_to(log_sigmoid(-z), rd), eps), rd);
        f.loss = type == AA_DPO_SIGMOID ? round_to(m1 - m2, rd)
                                        : round_to(__fmul_rn(round_to(m1 + m2, rd), 1.f / (1.f - 2.f * eps)), rd);
      }
      f.s0 = z;
      break;
    }
    case AA_DPO_HINGE: {
      const float u = round_to(1.f - round_to(__fmul_rn(beta, round_to(a - b, rd)), rd), rd);
      f.loss = (u > 0.f || u != u) ? u : 0.f;
      f.s0 = f.loss;
      break;
    }
    case AA_DPO_IPO: {
      const float d = round_to(round_to(a - b, rd) - c, rd);
      f.loss = round_to(__fmul_rn(d, d), rd);
      f.s0 = d;
      break;
    }
    case AA_DPO_SPPO_HARD: {
      const float d1 = round_to(a - c, rd), d2 = round_to(b + c, rd);
      f.loss = round_to(round_to(__fmul_rn(d1, d1), rd) + round_to(__fmul_rn(d2, d2), rd), rd);
      f.s0 = d1;
      f.s1 = d2;
      break;
    }
    case AA_DPO_NCA_PAIR: {
      const float za = round_to(__fmul_rn(beta, a), rd), zb = round_to(__fmul_rn(beta, b), rd);
      const float t1 = round_to(log_sigmoid(za), rd), t2 = round_to(log_sigmoid(-za), rd);
      const float t3 = round_to(log_sigmoid(-zb), rd);
      f.loss = round_to(round_to(-t1 - __fmul_rn(0.5f, t2), rd) - __fmul_rn(0.5f, t3), rd);
      f.s0 = za;
      f.s1 = zb;
      break;
    }
    case AA_DPO_APO_ZERO: {
      const float sa = round_to(sigmoid_f(round_to(__fmul_rn(beta, a), rd)), rd);
      const float sb = round_to(sigmoid_f(round_to(__fmul_rn(beta, b), rd)), rd);
      f.loss = round_to(round_to(1.f - sa, rd) + sb, rd);
      f.s0 = sa;
      f.s1 = sb;
      break;
    }
    default: {  // AA_DPO_APO_DOWN
      const float sa = round_to(sigmoid_f(round_to(__fmul_rn(beta, a), rd)), rd);
      const float sh = round_to(sigmoid_f(round_to(__fmul_rn(beta, round_to(a - b, rd)), rd)), rd);
      f.loss = round_to(sa + round_to(1.f - sh, rd), rd);
      f.s0 = sa;
      f.s1 = sh;
      break;
    }
  }
  return f;
}

// sigmoid_backward(g, s) = g * (1 - s) * s, evaluated by ATen CUDA in the tensor's dtype: a rounding after each op
__device__ __forceinline__ float dsigmoid(float g, float s, int rd) {
  return round_to(__fmul_rn(round_to(__fmul_rn(g, round_to(1.f - s, rd)), rd), s), rd);
}

// d (gl * loss) / d (chosen sum, rejected sum) from the forward's (s0, s1); gl = d mean / d loss_i.  inv_nc / inv_nr:
// 1 / row count (IPO only).
__device__ __forceinline__ float2 dpo_obj_backward(int type, float gl, float s0, float s1, float beta, float eps,
                                                   float inv_nc, float inv_nr, int rd) {
  switch (type) {
    case AA_DPO_SIGMOID:
    case AA_DPO_ROBUST: {
      float gz;
      if (eps == 0.f) {
        gz = round_to(__fmul_rn(-gl, dlog_sigmoid(s0)), rd);
      } else {
        const float g0 = type == AA_DPO_ROBUST ? round_to(__fmul_rn(gl, 1.f / (1.f - 2.f * eps)), rd) : gl;
        const float dt1 = -round_to(__fmul_rn(g0, 1.f - eps), rd);
        const float dt2 = round_to(__fmul_rn(type == AA_DPO_ROBUST ? g0 : -g0, eps), rd);
        gz = round_to(round_to(__fmul_rn(dt1, dlog_sigmoid(s0)), rd) - round_to(__fmul_rn(dt2, dlog_sigmoid(-s0)), rd),
                      rd);
      }
      const float gh = round_to(__fmul_rn(gz, beta), rd);
      return make_float2(gh, -gh);
    }
    case AA_DPO_HINGE: {  // ReluBackward: no gradient where the result is <= 0
      const float gh = round_to(__fmul_rn(s0 > 0.f || s0 != s0 ? -gl : 0.f, beta), rd);
      return make_float2(gh, -gh);
    }
    case AA_DPO_IPO: {
      const float gd = round_to(__fmul_rn(gl, 2.f * s0), rd);
      return make_float2(round_to(__fmul_rn(gd, inv_nc), rd), round_to(__fmul_rn(-gd, inv_nr), rd));
    }
    case AA_DPO_SPPO_HARD:
      return make_float2(round_to(__fmul_rn(gl, 2.f * s0), rd), round_to(__fmul_rn(gl, 2.f * s1), rd));
    case AA_DPO_NCA_PAIR: {
      const float hg = __fmul_rn(-gl, 0.5f);
      const float gza = round_to(round_to(__fmul_rn(-gl, dlog_sigmoid(s0)), rd) -
                                     round_to(__fmul_rn(hg, dlog_sigmoid(-s0)), rd), rd);
      const float gzb = -round_to(__fmul_rn(hg, dlog_sigmoid(-s1)), rd);
      return make_float2(round_to(__fmul_rn(gza, beta), rd), round_to(__fmul_rn(gzb, beta), rd));
    }
    case AA_DPO_APO_ZERO:
      return make_float2(round_to(__fmul_rn(dsigmoid(-gl, s0, rd), beta), rd),
                         round_to(__fmul_rn(dsigmoid(gl, s1, rd), beta), rd));
    default: {  // AA_DPO_APO_DOWN
      const float gh = round_to(__fmul_rn(dsigmoid(-gl, s1, rd), beta), rd);
      const float ga = round_to(__fmul_rn(dsigmoid(gl, s0, rd), beta), rd);
      return make_float2(round_to(ga + gh, rd), -gh);
    }
  }
}

// ---- K2 extended objective: f-divergences, EXO, DiscoPOP and AOT (DESIGN section 4.13) -----------------------------
// Each restates tests/dpo_ext_port.py op for op, with the conventions of the objective variant above.  The
// per-pair thread keeps (a, b) in grad_seg and the last block re-runs the pair's forward next to its backward; AOT
// keeps its two sort keys there instead and is sorted, and its loss formed, by the last block.
struct DpoExtParams : DpoObjParams {
  int fdiv;       // AA_DPO_FDIV_*
  float f_alpha;  // alpha-divergence coefficient
  float tau;      // DiscoPOP temperature
  float exp_cap;  // cap_exp's clamp, floor(log(finfo(log-prob dtype).max) * 1e4) / 1e4
  float exo_c1, exo_c2;  // EXO's log(1 - e') and log(e'), formed by the caller in double and rounded to fp32 once
};

// ATen softplus (beta 1, threshold 20) and its backward g * z / (z + 1), z = exp(x), each in fp32 and rounded once
__device__ __forceinline__ float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float dsoftplus(float g, float x, int rd) {
  const float z = expf(x);
  return round_to(x > 20.f ? g : __fdiv_rn(__fmul_rn(g, z), z + 1.f), rd);
}

// exp(clamp(x, max = cap)): clamp passes NaN through and rounds its fp32 result
__device__ __forceinline__ float cap_exp(float x, float cap, int rd) {
  return round_to(expf(round_to(x != x ? x : fminf(x, cap), rd)), rd);
}

// h from a and b under the f-divergence
__device__ __forceinline__ float fdiv_forward(const DpoExtParams &p, float a, float b, int rd) {
  if (p.fdiv == AA_DPO_FDIV_ALPHA) {
    const float eb = cap_exp(round_to(__fmul_rn(b, -p.f_alpha), rd), p.exp_cap, rd);
    const float ea = cap_exp(round_to(__fmul_rn(a, -p.f_alpha), rd), p.exp_cap, rd);
    return round_to(__fmul_rn(round_to(eb - ea, rd), 1.f / p.f_alpha), rd);
  }
  const float h = round_to(a - b, rd);
  if (p.fdiv == AA_DPO_FDIV_JS) return round_to(h - round_to(round_to(softplus_f(a), rd) - round_to(softplus_f(b), rd), rd), rd);
  return h;
}

// (d / d a, d / d b) from d / d h.  Alpha: ExpBackward (grad * result), then no gradient where the clamp is active.
__device__ __forceinline__ float2 fdiv_backward(const DpoExtParams &p, float gh, float a, float b, int rd) {
  if (p.fdiv == AA_DPO_FDIV_ALPHA) {
    const float gd = round_to(__fmul_rn(gh, 1.f / p.f_alpha), rd);
    const float ta = round_to(__fmul_rn(a, -p.f_alpha), rd), tb = round_to(__fmul_rn(b, -p.f_alpha), rd);
    const float gta = ta <= p.exp_cap ? round_to(__fmul_rn(-gd, cap_exp(ta, p.exp_cap, rd)), rd) : 0.f;
    const float gtb = tb <= p.exp_cap ? round_to(__fmul_rn(gd, cap_exp(tb, p.exp_cap, rd)), rd) : 0.f;
    return make_float2(round_to(__fmul_rn(gta, -p.f_alpha), rd), round_to(__fmul_rn(gtb, -p.f_alpha), rd));
  }
  if (p.fdiv == AA_DPO_FDIV_JS)  // h = a - b and softplus(a) both reach a: two terms, added once
    return make_float2(round_to(gh + dsoftplus(-gh, a, rd), rd), round_to(-gh + dsoftplus(gh, b, rd), rd));
  return make_float2(gh, -gh);
}

// EXO (pair form) and DiscoPOP of h: (loss, d (gl * loss) / d h).  z reaches the loss along three paths; autograd adds
// their gradients in the order its engine runs them (the latest-created node first), so the sums below follow it.
__device__ __forceinline__ float2 exo_discopop(const DpoExtParams &p, float h, float gl, int rd) {
  const float z = round_to(__fmul_rn(p.beta, h), rd);
  if (p.loss_type == AA_DPO_EXO_PAIR) {
    const float c1 = p.exo_c1, c2 = p.exo_c2;
    const float s1 = round_to(sigmoid_f(z), rd), t1 = round_to(round_to(log_sigmoid(z), rd) - c1, rd);
    const float s2 = round_to(sigmoid_f(-z), rd), t2 = round_to(round_to(log_sigmoid(-z), rd) - c2, rd);
    const float loss = round_to(round_to(__fmul_rn(s1, t1), rd) + round_to(__fmul_rn(s2, t2), rd), rd);
    const float g_nz = round_to(round_to(__fmul_rn(round_to(__fmul_rn(gl, s2), rd), dlog_sigmoid(-z)), rd) +
                                    dsigmoid(round_to(__fmul_rn(gl, t2), rd), s2, rd), rd);
    const float g_l1 = round_to(__fmul_rn(round_to(__fmul_rn(gl, s1), rd), dlog_sigmoid(z)), rd);
    const float gz = round_to(round_to(-g_nz + g_l1, rd) + dsigmoid(round_to(__fmul_rn(gl, t1), rd), s1, rd), rd);
    return make_float2(loss, round_to(__fmul_rn(gz, p.beta), rd));
  }
  // AA_DPO_DISCOPOP: m = sigmoid(z / tau), loss = -logsigmoid(z) * (1 - m) + exp(-z) * m
  const float inv_tau = 1.f / p.tau;
  const float m = round_to(sigmoid_f(round_to(__fmul_rn(z, inv_tau), rd)), rd);
  const float lc = -round_to(log_sigmoid(z), rd), ec = round_to(expf(-z), rd), om = round_to(1.f - m, rd);
  const float loss = round_to(round_to(__fmul_rn(lc, om), rd) + round_to(__fmul_rn(ec, m), rd), rd);
  const float gm = round_to(round_to(__fmul_rn(gl, ec), rd) - round_to(__fmul_rn(gl, lc), rd), rd);
  const float g_e = -round_to(__fmul_rn(round_to(__fmul_rn(gl, m), rd), ec), rd);
  const float g_l = round_to(__fmul_rn(-round_to(__fmul_rn(gl, om), rd), dlog_sigmoid(z)), rd);
  const float g_t = round_to(__fmul_rn(dsigmoid(gm, m, rd), inv_tau), rd);
  const float gz = round_to(round_to(g_e + g_l, rd) + g_t, rd);
  return make_float2(loss, round_to(__fmul_rn(gz, p.beta), rd));
}

__device__ __forceinline__ bool dpo_aot(int type) { return type == AA_DPO_AOT || type == AA_DPO_AOT_PAIR; }
// the types and f-divergences aa_dpo_loss_obj already has: the same arithmetic, the same stored operands
__device__ __forceinline__ bool dpo_obj_arith(const DpoExtParams &p) {
  return p.loss_type <= AA_DPO_APO_DOWN && p.fdiv == AA_DPO_FDIV_REVERSE_KL;
}

// A pair of a non-AOT new type or f-divergence: (loss, d (gl * loss) / d a, d (gl * loss) / d b)
__device__ __forceinline__ float3 dpo_ext_pair(const DpoExtParams &p, float a, float b, float gl, int rd) {
  const float h = fdiv_forward(p, a, b, rd);
  float2 r;
  if (p.loss_type == AA_DPO_EXO_PAIR || p.loss_type == AA_DPO_DISCOPOP) {
    r = exo_discopop(p, h, gl, rd);
  } else {  // SIGMOID / ROBUST / HINGE of the f-divergence's h: a = h, b = 0 makes their h - 0 = h exactly
    const DpoPairFwd f = dpo_obj_forward(p.loss_type, h, 0.f, p.beta, p.eps, rd);
    r = make_float2(f.loss, dpo_obj_backward(p.loss_type, gl, f.s0, f.s1, p.beta, p.eps, 0.f, 0.f, rd).x);
  }
  const float2 g = fdiv_backward(p, r.y, a, b, rd);
  return make_float3(r.x, g.x, g.y);
}

// The per-pair thread: the loss and the two operands the last block reads back (AOT: its sort keys, loss 0 for now)
__device__ __forceinline__ DpoPairFwd dpo_ext_forward(const DpoExtParams &p, float a, float b, float pc, float pr,
                                                      float rc, float rr, int rd) {
  if (p.loss_type == AA_DPO_AOT) return DpoPairFwd{0.f, round_to(pc - pr, rd), round_to(rc - rr, rd)};
  if (p.loss_type == AA_DPO_AOT_PAIR) return DpoPairFwd{0.f, a, b};
  if (dpo_obj_arith(p)) return dpo_obj_forward(p.loss_type, a, b, p.beta, p.eps, rd);
  return DpoPairFwd{dpo_ext_pair(p, a, b, 0.f, rd).x, a, b};
}

// AOT in the last block: a stable rank sort of the kept pairs' two keys (torch.sort(stable=True): NaN last, ties to the
// smaller pair index), exact and deterministic; then delta_k = key1_(k) - key2_(k) and the sigmoid loss of each
// position k.  per_pair[0][i] becomes the loss at the position of pair i's first key.
struct DpoAotSmem {
  float key1[AA_DPO_AOT_MAX_PAIRS], key2[AA_DPO_AOT_MAX_PAIRS];
  float pos[AA_DPO_AOT_MAX_PAIRS];  // the sorted second keys, then z = beta * delta_k at each position k
  int rank1[AA_DPO_AOT_MAX_PAIRS], rank2[AA_DPO_AOT_MAX_PAIRS];  // -1: a skipped pair
  unsigned char keep[AA_DPO_AOT_MAX_PAIRS];
};
__device__ __forceinline__ DpoAotSmem &dpo_aot_smem() {
  __shared__ DpoAotSmem s;
  return s;
}

__device__ __forceinline__ bool sorts_before(float xj, int j, float xi, int i) {
  if (xi != xi) return xj == xj || j < i;
  if (xj != xj) return false;
  return xj < xi || (xj == xi && j < i);
}

template <int THREADS>
__device__ void dpo_aot_sort(const DpoExtParams &p) {
  DpoAotSmem &s = dpo_aot_smem();
  const int B = p.n_pairs, rd = p.round_dt, tid = threadIdx.x;
  const volatile float *v_key = p.grad_seg, *v_valid = p.per_pair + 4 * B;
  for (int k = tid; k < B; k += THREADS) {
    s.key1[k] = v_key[k];
    s.key2[k] = v_key[B + k];
    s.keep[k] = v_valid[k] != 0.f;
  }
  __syncthreads();
  for (int i = tid; i < B; i += THREADS) {
    int r1 = -1, r2 = -1;
    if (s.keep[i]) {
      r1 = r2 = 0;
      const float x1 = s.key1[i], x2 = s.key2[i];
      for (int j = 0; j < B; ++j) {
        if (s.keep[j]) {
          r1 += sorts_before(s.key1[j], j, x1, i);
          r2 += sorts_before(s.key2[j], j, x2, i);
        }
      }
    }
    s.rank1[i] = r1;
    s.rank2[i] = r2;
  }
  __syncthreads();
  for (int i = tid; i < B; i += THREADS)
    if (s.rank2[i] >= 0) s.pos[s.rank2[i]] = s.key2[i];
  __syncthreads();
  for (int i = tid; i < B; i += THREADS) {
    const int k = s.rank1[i];
    if (k >= 0) {  // position k is read and rewritten by this thread alone (the ranks are a permutation)
      const DpoPairFwd f = dpo_obj_forward(AA_DPO_SIGMOID, round_to(s.key1[i] - s.pos[k], rd), 0.f, p.beta, p.eps, rd);
      p.per_pair[i] = f.loss;
      s.pos[k] = f.s0;
    }
  }
  __syncthreads();
}

// (d / d chosen sum, d / d rejected sum) of a kept pair k of the extended variant; s0, s1: what its forward stored
__device__ __forceinline__ float2 dpo_ext_backward(const DpoExtParams &p, int k, float gl, float s0, float s1,
                                                   float inv_nc, float inv_nr, int rd) {
  if (dpo_aot(p.loss_type)) {  // SortBackward: each key takes the gradient of the position it landed in
    const DpoAotSmem &s = dpo_aot_smem();
    const float g1 = dpo_obj_backward(AA_DPO_SIGMOID, gl, s.pos[s.rank1[k]], 0.f, p.beta, p.eps, 0.f, 0.f, rd).x;
    if (p.loss_type == AA_DPO_AOT) return make_float2(g1, -g1);  // key1 = pc - pr
    return make_float2(g1, -dpo_obj_backward(AA_DPO_SIGMOID, gl, s.pos[s.rank2[k]], 0.f, p.beta, p.eps, 0.f, 0.f, rd).x);
  }
  if (dpo_obj_arith(p)) return dpo_obj_backward(p.loss_type, gl, s0, s1, p.beta, p.eps, inv_nc, inv_nr, rd);
  const float3 r = dpo_ext_pair(p, s0, s1, gl, rd);
  return make_float2(r.y, r.z);
}

// The last block of the objective variant, after the metric means: the RPO NLL term (alpha > 0), then the seeds.
// per_pair[3] holds each pair's chosen sum and grad_seg the forward's (s0, s1) until they are replaced here.
template <int THREADS, class Params>
__device__ __forceinline__ void dpo_obj_finish(const Params &p, float sum_loss_over_n, float inv_n, float *scratch) {
  const int B = p.n_pairs, rd = p.round_dt, tid = threadIdx.x;
  volatile float *v_g = p.per_pair + 3 * B, *v_seg = p.grad_seg;
  const volatile float *v_valid = p.per_pair + 4 * B;
  float g_nll = 0.f;
  if (p.alpha > 0.f) {  // NLL = -(sum of the kept chosen sums) / (their scored rows): the token mean, as in RPO
    // the count is summed in integers and rounded to fp32 once, as ATen converts the reference's exact Python count:
    // an fp32 sum past 2^24 rounds at every level of the tree
    __shared__ unsigned long long cnt_total;
    if (tid == 0) cnt_total = 0ull;
    float s_pc = 0.f;
    long long s_cnt = 0;
    for (int k = tid; k < B; k += THREADS) {
      if (v_valid[k] != 0.f) {
        s_pc += v_g[k];
        s_cnt += p.counts[k];
      }
    }
    s_pc = block_sum<THREADS>(s_pc, scratch);  // its barriers order the zeroing above before the adds below
    atomicAdd(&cnt_total, static_cast<unsigned long long>(s_cnt));
    __syncthreads();
    const float inv_cnt = 1.f / static_cast<float>(static_cast<long long>(cnt_total));  // x / int: x * (1 / n)
    const float nll = -round_to(__fmul_rn(round_to(s_pc, rd), inv_cnt), rd);
    g_nll = round_to(__fmul_rn(-round_to(p.alpha, rd), inv_cnt), rd);  // Add -> Mul(alpha) -> Neg -> Div -> Sum
    if (tid == 0) {
      p.stats[0] = round_to(round_to(sum_loss_over_n, rd) + round_to(__fmul_rn(nll, p.alpha), rd), rd);
      p.stats[8] = nll;
    }
  }
  const float gl = round_to(inv_n, rd);  // MeanBackward
  for (int k = tid; k < B; k += THREADS) {
    float gc = 0.f, gr = -0.f;  // a skipped pair: the seeds aa_dpo_loss writes (+0, -0)
    if (v_valid[k] != 0.f) {
      const bool ipo = p.loss_type == AA_DPO_IPO;
      float2 g;
      if constexpr (std::is_same<Params, DpoExtParams>::value)
        g = dpo_ext_backward(p, k, gl, v_seg[k], v_seg[B + k], ipo ? 1.f / static_cast<float>(p.counts[k]) : 0.f,
                             ipo ? 1.f / static_cast<float>(p.counts[B + k]) : 0.f, rd);
      else
        g = dpo_obj_backward(p.loss_type, gl, v_seg[k], v_seg[B + k], p.beta, p.eps,
                             ipo ? 1.f / static_cast<float>(p.counts[k]) : 0.f,
                             ipo ? 1.f / static_cast<float>(p.counts[B + k]) : 0.f, rd);
      gc = p.alpha > 0.f ? round_to(g.x + g_nll, rd) : g.x;
      gr = g.y;
    }
    v_g[k] = gc;
    v_seg[k] = gc;
    v_seg[B + k] = gr;
  }
}

template <int THREADS, class Params>
__global__ void __launch_bounds__(THREADS) dpo_loss_kernel(const Params p) {
  constexpr bool OBJ = std::is_base_of<DpoObjParams, Params>::value;
  constexpr bool EXT = std::is_same<Params, DpoExtParams>::value;
  __shared__ float scratch[33];
  __shared__ int same_flag;
  const int i = blockIdx.x, tid = threadIdx.x;
  const int B = p.n_pairs;
  const int rd = p.round_dt;
  float *loss_i = p.per_pair, *better_i = p.per_pair + B, *worse_i = p.per_pair + 2 * B,
        *g_i = p.per_pair + 3 * B, *valid_i = p.per_pair + 4 * B;

  const float pc = round_to(row_sum<THREADS>(p.policy_lp, p.lp_dtype, int64_t(i) * p.row_stride, p.width, scratch), rd);
  const float pr = round_to(row_sum<THREADS>(p.policy_lp, p.lp_dtype, int64_t(B + i) * p.row_stride, p.width, scratch), rd);
  float rc = 0.f, rr = 0.f;  // reference-free (OBJ with ref_lp == NULL): the reference sums are 0
  if (!OBJ || p.ref_lp) {
    rc = round_to(row_sum<THREADS>(p.ref_lp, p.lp_dtype, int64_t(i) * p.row_stride, p.width, scratch), rd);
    rr = round_to(row_sum<THREADS>(p.ref_lp, p.lp_dtype, int64_t(B + i) * p.row_stride, p.width, scratch), rd);
  }

  bool valid = true;
  if (p.ids) {  // text_audio_to_text/dpo.py:138: skip when chosen ids == rejected ids
    if (tid == 0) same_flag = 1;
    __syncthreads();
    const int64_t *a = p.ids + int64_t(i) * p.ids_row_stride;
    const int64_t *b = p.ids + int64_t(B + i) * p.ids_row_stride;
    bool diff = false;
    for (int k = tid; k < p.L; k += THREADS) diff |= (a[k] != b[k]);
    if (diff) same_flag = 0;
    __syncthreads();
    valid = (same_flag == 0);
  }

  if (tid == 0) {
    const float ratio_c = round_to(pc - rc, rd);
    const float ratio_r = round_to(pr - rr, rd);
    if constexpr (OBJ) {
      float a = ratio_c, b = ratio_r;
      if (p.loss_type == AA_DPO_IPO) {  // the four sums divided by their row counts first (x / int: x * (1 / n))
        const float inv_c = 1.f / static_cast<float>(p.counts[i]), inv_r = 1.f / static_cast<float>(p.counts[B + i]);
        a = round_to(round_to(__fmul_rn(pc, inv_c), rd) - round_to(__fmul_rn(rc, inv_c), rd), rd);
        b = round_to(round_to(__fmul_rn(pr, inv_r), rd) - round_to(__fmul_rn(rr, inv_r), rd), rd);
      }
      DpoPairFwd f;
      if constexpr (EXT)
        f = dpo_ext_forward(p, a, b, pc, pr, rc, rr, rd);
      else
        f = dpo_obj_forward(p.loss_type, a, b, p.beta, p.eps, rd);
      loss_i[i] = f.loss;
      better_i[i] = round_to(p.beta * ratio_c, rd);  // the metrics keep the summed ratios for every loss type
      worse_i[i] = round_to(p.beta * ratio_r, rd);
      g_i[i] = pc;  // the chosen sum, for the NLL term; the last block overwrites it with the chosen seed
      p.grad_seg[i] = f.s0;  // the backward's operands, until the last block turns them into the seeds
      p.grad_seg[B + i] = f.s1;
    } else {
      const float z = round_to(p.beta * round_to(ratio_c - ratio_r, rd), rd);
      loss_i[i] = -round_to(log_sigmoid(z), rd);
      better_i[i] = round_to(p.beta * ratio_c, rd);
      worse_i[i] = round_to(p.beta * ratio_r, rd);
      g_i[i] = z;  // converted to the gradient coefficient by the last block
    }
    valid_i[i] = valid ? 1.f : 0.f;
  }

  if (!last_block_arrives(p.counter, gridDim.x)) return;
  if constexpr (EXT) {
    if (dpo_aot(p.loss_type)) dpo_aot_sort<THREADS>(p);
  }

  // ---- final reduction over pairs (fixed order -> deterministic) ----
  // other blocks' results: read through volatile so no stale L1 line can be used
  const volatile float *v_loss = loss_i, *v_better = better_i, *v_worse = worse_i, *v_valid = valid_i;
  volatile float *v_g = g_i;
  float n = 0.f, s_loss = 0.f, s_rew = 0.f, s_bet = 0.f, s_wor = 0.f, s_acc = 0.f, s_mar = 0.f;
  for (int k = tid; k < B; k += THREADS) {
    if (v_valid[k] != 0.f) {
      const float b = v_better[k], w = v_worse[k];
      n += 1.f;
      s_loss += v_loss[k];
      s_bet += b;
      s_wor += w;
      s_rew += round_to(b + w, rd);
      s_mar += round_to(b - w, rd);
      s_acc += (b > w) ? 1.f : 0.f;
    }
  }
  n = block_sum<THREADS>(n, scratch);
  s_loss = block_sum<THREADS>(s_loss, scratch);
  s_rew = block_sum<THREADS>(s_rew, scratch);
  s_bet = block_sum<THREADS>(s_bet, scratch);
  s_wor = block_sum<THREADS>(s_wor, scratch);
  s_acc = block_sum<THREADS>(s_acc, scratch);
  s_mar = block_sum<THREADS>(s_mar, scratch);
  const float inv_n = 1.f / n;
  if (tid == 0) {
    p.stats[0] = round_to(s_loss * inv_n, rd);
    p.stats[1] = round_to(s_rew * inv_n, rd);
    p.stats[2] = round_to(s_bet * inv_n, rd);
    p.stats[3] = round_to(s_wor * inv_n, rd);
    p.stats[4] = s_acc * inv_n;  // (better > worse).float().mean() is fp32 in the reference
    p.stats[5] = round_to(s_mar * inv_n, rd);
    p.stats[6] = n;
    // the sticky status word rides in the free lane: the trainers read it with the metrics (no extra sync) and raise
    p.stats[7] = p.status ? static_cast<float>(*reinterpret_cast<const volatile int32_t *>(p.status)) : 0.f;
  }
  if constexpr (OBJ) {
    dpo_obj_finish<THREADS, Params>(p, s_loss * inv_n, inv_n, scratch);
    return;
  }
  if (p.coll.world > 1 && p.stats_global) {
    // the packed-metric all-reduce of train_step (trainers/text_to_text/dpo.py:222-227), done by this very
    // block over NVLink peer memory: one kernel computes the loss AND its collective
    __syncthreads();  // p.stats written by thread 0 above
    __threadfence();
    p2p_allreduce_packed(p.coll, p.stats, p.stats_global, 8);
  }
  // upstream gradient of the mean loss w.r.t. each sequence log-prob sum (autograd chain:
  // MeanBackward -> NegBackward -> LogSigmoidBackward -> MulBackward(beta) -> SubBackward)
  const float gl = round_to(inv_n, rd);
  for (int k = tid; k < B; k += THREADS) {
    float g = 0.f;
    if (v_valid[k] != 0.f) {
      const float gz = round_to(-gl * dlog_sigmoid(v_g[k]), rd);
      g = round_to(gz * p.beta, rd);
    }
    v_g[k] = g;
    if (p.grad_seg) {
      p.grad_seg[k] = g;
      p.grad_seg[B + k] = -g;
    }
  }
}

// ---- pair bookkeeping of SimPO / ORPO / KTO (SURVEY 8f row 2) ---------------------------------------------
// trainers/text_to_text/simpo.py:63-77 (same block in orpo.py:63-77, kto.py:113-125): per pair, a Python loop with
// 4 host syncs in the reference -- identical-pair test, last attended index of both rows, first index where the
// two id rows diverge.  Integer, bit-exact.  out = int32 [4][n_pairs]: valid, diverge_index, end_better, end_worse.
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
    pair_slices_kernel(const int64_t *__restrict__ ids, int64_t ids_stride, const void *__restrict__ mask, int mask_kind,
                       int64_t mask_stride, int B, int L, int32_t *__restrict__ out, int32_t *status) {
  __shared__ int sh_div, sh_ec, sh_er;
  const int i = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) {
    sh_div = L;
    sh_ec = -1;
    sh_er = -1;
  }
  __syncthreads();
  const int64_t *a = ids + static_cast<int64_t>(i) * ids_stride;
  const int64_t *b = ids + static_cast<int64_t>(B + i) * ids_stride;
  int dv = L, ec = -1, er = -1;
  for (int k = tid; k < L; k += THREADS) {
    if (a[k] != b[k]) dv = min(dv, k);
    const bool mc = (mask_kind == AA_MASK_U8) ? reinterpret_cast<const uint8_t *>(mask)[i * mask_stride + k] != 0
                                              : reinterpret_cast<const int64_t *>(mask)[i * mask_stride + k] != 0;
    const bool mr = (mask_kind == AA_MASK_U8) ? reinterpret_cast<const uint8_t *>(mask)[(B + i) * mask_stride + k] != 0
                                              : reinterpret_cast<const int64_t *>(mask)[(B + i) * mask_stride + k] != 0;
    if (mc) ec = max(ec, k);
    if (mr) er = max(er, k);
  }
  if (dv < L) atomicMin(&sh_div, dv);
  if (ec >= 0) atomicMax(&sh_ec, ec);
  if (er >= 0) atomicMax(&sh_er, er);
  __syncthreads();
  if (tid == 0) {
    const bool valid = sh_div < L;  // identical id rows are skipped (simpo.py:61-62)
    out[i] = valid ? 1 : 0;
    out[B + i] = valid ? sh_div : 0;
    out[2 * B + i] = sh_ec;
    out[3 * B + i] = sh_er;
    // only a valid pair raises: the reference skips an identical pair before it reads either mask row
    if (status && valid) {
      if (sh_ec < 0 || sh_er < 0) atomicOr(status, AA_STATUS_EMPTY_MASK);
      else if (sh_div > sh_ec || sh_div > sh_er) atomicOr(status, AA_STATUS_DIVERGE_RANGE);  // the asserts
    }
  }
}

// sums[r] = sum(lp[r, lo : min(hi, W)]) for r < 2B: lo = diverge[r mod B], hi = end_better[r]+1 / end_worse[r-B]+1
// (Python slice semantics: an empty or out-of-range slice sums to 0); rounded to the lp dtype in FAITHFUL mode.
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
    slice_sums_kernel(const void *lp, int dtype, int64_t row_stride, int B, int W, const int32_t *__restrict__ slices,
                      int round_dt, float *__restrict__ sums) {
  __shared__ float scratch[33];
  const int r = blockIdx.x;
  const int i = r % B;
  const int lo = slices[B + i];
  const int hi = min(((r < B) ? slices[2 * B + i] : slices[3 * B + i]) + 1, W);
  float acc = 0.f;
  for (int k = lo + threadIdx.x; k < hi; k += THREADS) acc += load_as_float(lp, r * row_stride + k, dtype);
  acc = block_sum<THREADS>(acc, scratch);
  if (threadIdx.x == 0) sums[r] = round_to(acc, round_dt);
}

// ---- reward-model pairwise loss (SURVEY 8f row 2: sibling loss reusing K3) --------------------------------
// trainers/text_to_text/rm.py:97-132: loss = mean(-logsigmoid(higher_end - lower_end))
//                                            [+ regularization * mean(square(stack([lower, higher])))]
// end_scores are always fp32 in the reference (models/llama.py:63 `.float()`), so this is plain fp32.
// One CTA: forward, accuracy AND d loss / d end_scores in the same launch.
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
    rm_pair_loss_kernel(const float *__restrict__ end_scores, int B, float reg, float *out, float *__restrict__ grad) {
  __shared__ float scratch[33];
  float s_loss = 0.f, s_sq = 0.f, s_acc = 0.f;
  const float inv_b = 1.f / static_cast<float>(B);
  for (int i = threadIdx.x; i < B; i += THREADS) {
    const float h = end_scores[i], l = end_scores[B + i];
    const float z = h - l;
    s_loss += -log_sigmoid(z);
    s_sq += h * h + l * l;
    s_acc += (h > l) ? 1.f : 0.f;
    if (grad) {
      const float ds = -dlog_sigmoid(z) * inv_b;  // d mean(-logsigmoid(z)) / dz
      const float r = (reg > 0.f) ? reg * inv_b : 0.f;  // d (reg * mean over 2B of x^2) / dx = reg * x / B
      grad[i] = ds + r * h;
      grad[B + i] = -ds + r * l;
    }
  }
  s_loss = block_sum<THREADS>(s_loss, scratch);
  s_sq = block_sum<THREADS>(s_sq, scratch);
  s_acc = block_sum<THREADS>(s_acc, scratch);
  if (threadIdx.x == 0) {
    float loss = s_loss * inv_b;
    if (reg > 0.f) loss += reg * (s_sq * 0.5f * inv_b);
    out[0] = loss;
    out[1] = s_acc * inv_b;
  }
}

// ---- cost-model pairwise loss (Safe RLHF's cost model; sibling of the RM loss) -----------------------------
// trainers/text_to_text/cost_model.py:97-144, with h / l the higher- / lower-cost end scores (dtype E):
//   cost   = -mean(logsigmoid(h * sb)) - mean(logsigmoid(l * sw))      sb / sw: is_better_safe / is_worse_safe
//   loss   = scale * cost - mean(logsigmoid(h - l)) [+ reg * mean(square(stack([l, h])))]
// The signs arrive cast to their product dtype Pb = result_type(h, sb) (E or fp32), likewise Pw; the cost and the
// loss are then in Pc = promote(Pb, Pw).  FAITHFUL rounds to E / Pb / Pw / Pc wherever the eager ops round; every
// product is __fmul_rn so that no rounding point is contracted away.  One CTA: forward, accuracy AND d loss / d
// end_scores in the same launch.  A separate kernel from the RM loss: RM's arithmetic (fp32 only) stays as it is.
struct CostParams {
  const void *scores;
  const void *better_signs;
  const void *worse_signs;
  int score_dt, better_dt, worse_dt;
  int n_pairs;
  float scale, reg;
  int faithful;
  void *loss;     // 0-dim, dtype Pc
  float *stats;   // [loss, accuracy]
  void *grad;     // optional, [2B] in E
};

template <int THREADS>
__global__ void __launch_bounds__(THREADS) cost_pair_loss_kernel(const CostParams p) {
  __shared__ float scratch[33];
  const int B = p.n_pairs, E = p.score_dt;
  const int out_dt = (p.better_dt == AA_F32 || p.worse_dt == AA_F32) ? AA_F32 : E;
  const int re = p.faithful ? E : AA_F32, rb = p.faithful ? p.better_dt : AA_F32;
  const int rw = p.faithful ? p.worse_dt : AA_F32, rc = p.faithful ? out_dt : AA_F32;
  const float inv_b = 1.f / static_cast<float>(B), inv_2b = 1.f / static_cast<float>(2 * B);
  const bool use_reg = p.reg > 0.f;
  // autograd's chain from d loss = 1, each gradient cast to its input's dtype at the promotion points
  // (a mean's backward multiplies by the fp32 reciprocal of the count, as ATen CUDA divides by a scalar)
  const float g_cost = round_to(p.scale, rc);                                     // MulBackward(scale)
  const float g_lsb = round_to(__fmul_rn(-round_to(g_cost, rb), inv_b), rb);      // Sub -> Neg -> MeanBackward
  const float g_lsw = round_to(__fmul_rn(-round_to(g_cost, rw), inv_b), rw);      // Sub(other) -> MeanBackward
  const float g_lso = round_to(-inv_b, re);                                       // Neg -> MeanBackward
  const float g_sq = round_to(__fmul_rn(round_to(p.reg, re), inv_2b), re);        // MulBackward(reg) -> MeanBackward
  float s_b = 0.f, s_w = 0.f, s_o = 0.f, s_sq = 0.f, s_acc = 0.f;
  for (int i = threadIdx.x; i < B; i += THREADS) {
    const float h = load_as_float(p.scores, i, E), l = load_as_float(p.scores, B + i, E);
    const float sb = load_as_float(p.better_signs, i, p.better_dt), sw = load_as_float(p.worse_signs, i, p.worse_dt);
    const float hb = round_to(__fmul_rn(h, sb), rb), lw = round_to(__fmul_rn(l, sw), rw), z = round_to(h - l, re);
    s_b += round_to(log_sigmoid(hb), rb);
    s_w += round_to(log_sigmoid(lw), rw);
    s_o += round_to(log_sigmoid(z), re);
    s_sq += round_to(__fmul_rn(h, h), re) + round_to(__fmul_rn(l, l), re);
    s_acc += (h > l) ? 1.f : 0.f;
    if (p.grad) {
      // the engine adds the contributions in reverse order of creation: reg (stack), then h - l, then the cost term
      const float gz = round_to(__fmul_rn(g_lso, dlog_sigmoid(z)), re);
      float gh = gz, gl = -gz;
      if (use_reg) {
        gh = round_to(round_to(__fmul_rn(g_sq, round_to(2.f * h, re)), re) + gz, re);
        gl = round_to(round_to(__fmul_rn(g_sq, round_to(2.f * l, re)), re) - gz, re);
      }
      // MulBackward(h * sb): (grad * sb) in Pb, then cast to E
      const float ch = round_to(round_to(__fmul_rn(round_to(__fmul_rn(g_lsb, dlog_sigmoid(hb)), rb), sb), rb), re);
      const float cl = round_to(round_to(__fmul_rn(round_to(__fmul_rn(g_lsw, dlog_sigmoid(lw)), rw), sw), rw), re);
      store_from_float(p.grad, i, E, round_to(gh + ch, re));
      store_from_float(p.grad, B + i, E, round_to(gl + cl, re));
    }
  }
  s_b = block_sum<THREADS>(s_b, scratch);
  s_w = block_sum<THREADS>(s_w, scratch);
  s_o = block_sum<THREADS>(s_o, scratch);
  s_sq = block_sum<THREADS>(s_sq, scratch);
  s_acc = block_sum<THREADS>(s_acc, scratch);
  if (threadIdx.x == 0) {
    const float mb = round_to(__fmul_rn(s_b, inv_b), rb), mw = round_to(__fmul_rn(s_w, inv_b), rw);
    const float mo = round_to(__fmul_rn(s_o, inv_b), re);
    const float cost = round_to(-mb - mw, rc);
    float loss = round_to(round_to(__fmul_rn(p.scale, cost), rc) - mo, rc);
    if (use_reg) loss = round_to(loss + round_to(__fmul_rn(p.reg, round_to(__fmul_rn(s_sq, inv_2b), re)), re), rc);
    store_from_float(p.loss, 0, out_dt, loss);  // f32 mode: the fp32 result, rounded once to the reference's dtype
    p.stats[0] = loss;                          // f32 mode: unrounded
    p.stats[1] = s_acc * inv_b;  // (h > l).float().mean() is fp32 in the reference
  }
}

}  // namespace aa

using namespace aa;

extern "C" int aa_pair_slices(const int64_t *input_ids, int64_t ids_row_stride, const void *attention_mask,
                              int mask_kind, int64_t mask_row_stride, int32_t n_pairs, int32_t L, int32_t *out,
                              int32_t *status, void *stream) {
  AA_REQUIRE(n_pairs > 0 && L > 0 && input_ids && attention_mask && out, AA_ERR_ARG, "aa_pair_slices: bad arguments");
  pair_slices_kernel<256><<<n_pairs, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      input_ids, ids_row_stride, attention_mask, mask_kind, mask_row_stride, n_pairs, L, out, status);
  return check_launch("aa_pair_slices");
}

extern "C" int aa_slice_sums(const void *lp, int lp_dtype, int64_t lp_row_stride, int32_t n_pairs, int32_t width,
                             const int32_t *slices, int mode, float *sums, void *stream) {
  AA_REQUIRE(n_pairs > 0 && width >= 0 && lp && slices && sums, AA_ERR_ARG, "aa_slice_sums: bad arguments");
  slice_sums_kernel<128><<<2 * n_pairs, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      lp, lp_dtype, lp_row_stride, n_pairs, width, slices, mode == AA_MODE_FAITHFUL ? lp_dtype : AA_F32, sums);
  return check_launch("aa_slice_sums");
}

extern "C" int aa_rm_pair_loss(const float *end_scores, int32_t n_pairs, float regularization, float *out,
                               float *grad_end_scores, void *stream) {
  AA_REQUIRE(n_pairs > 0 && end_scores && out, AA_ERR_ARG, "aa_rm_pair_loss: bad arguments");
  rm_pair_loss_kernel<256><<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(end_scores, n_pairs, regularization, out,
                                                                            grad_end_scores);
  return check_launch("aa_rm_pair_loss");
}

extern "C" int aa_cost_pair_loss(const void *end_scores, int score_dtype, const void *better_signs, int better_dtype,
                                 const void *worse_signs, int worse_dtype, int32_t n_pairs, float scale_coeff,
                                 float regularization, int mode, void *loss, float *stats, void *grad_end_scores,
                                 void *stream) {
  AA_REQUIRE(n_pairs > 0, AA_ERR_ARG, "aa_cost_pair_loss: bad sizes");
  AA_REQUIRE(end_scores && better_signs && worse_signs && loss && stats, AA_ERR_ARG, "aa_cost_pair_loss: null pointer");
  AA_REQUIRE(score_dtype == AA_BF16 || score_dtype == AA_F16 || score_dtype == AA_F32, AA_ERR_DTYPE,
             "aa_cost_pair_loss: bad dtype %d", score_dtype);
  AA_REQUIRE((better_dtype == score_dtype || better_dtype == AA_F32) && (worse_dtype == score_dtype || worse_dtype == AA_F32),
             AA_ERR_DTYPE, "aa_cost_pair_loss: bad sign dtype %d / %d for end-score dtype %d", better_dtype, worse_dtype,
             score_dtype);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "aa_cost_pair_loss: bad mode %d", mode);
  const CostParams p{end_scores, better_signs, worse_signs, score_dtype, better_dtype, worse_dtype, n_pairs,
                     scale_coeff, regularization, mode == AA_MODE_FAITHFUL, loss, stats, grad_end_scores};
  cost_pair_loss_kernel<256><<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("aa_cost_pair_loss");
}

extern "C" int aa_strip_pad_tail(const int64_t *input_ids, int32_t n_samples, int32_t L,
                                 int64_t ids_row_stride, int64_t pad_id, int strip,
                                 const int32_t *response_lens, int64_t *labels_out, int64_t out_stride,
                                 int32_t *status, void *stream) {
  AA_REQUIRE(n_samples >= 0 && L > 0, AA_ERR_ARG, "aa_strip_pad_tail: bad sizes");
  if (n_samples == 0) return AA_OK;
  AA_REQUIRE(input_ids && response_lens && labels_out, AA_ERR_ARG, "aa_strip_pad_tail: null pointer");
  strip_pad_tail_kernel<256><<<n_samples, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      input_ids, L, ids_row_stride, pad_id, strip, response_lens, labels_out, out_stride, status);
  return check_launch("aa_strip_pad_tail");
}

extern "C" int aa_dpo_loss(const void *policy_lp, const void *ref_lp, int lp_dtype, int32_t n_pairs,
                           int32_t width, int64_t lp_row_stride, float scale_coeff, int mode,
                           const int64_t *input_ids, int32_t L, int64_t ids_row_stride,
                           float *per_pair, float *grad_seg, float *stats, uint32_t *counter,
                           const aa_coll *coll, float *stats_global, const int32_t *status, void *stream) {
  AA_REQUIRE(n_pairs > 0 && width >= 0, AA_ERR_ARG, "aa_dpo_loss: bad sizes");
  AA_REQUIRE(policy_lp && ref_lp && per_pair && stats && counter, AA_ERR_ARG, "aa_dpo_loss: null pointer");
  AA_REQUIRE(lp_dtype == AA_BF16 || lp_dtype == AA_F16 || lp_dtype == AA_F32, AA_ERR_DTYPE,
             "aa_dpo_loss: bad dtype %d", lp_dtype);
  DpoParams p{policy_lp, ref_lp, lp_dtype, n_pairs, width, lp_row_stride, scale_coeff,
              mode == AA_MODE_FAITHFUL ? lp_dtype : AA_F32, input_ids, L, ids_row_stride,
              per_pair, grad_seg, stats, counter, stats_global, CollParams{nullptr, 0, 1, 0u, 0u}, status};
  if (coll && coll->world > 1) {
    AA_REQUIRE(coll->peer_bufs && stats_global && coll->world <= 32 && coll->rank >= 0 && coll->rank < coll->world,
               AA_ERR_ARG, "aa_dpo_loss: bad collective descriptor");
    p.coll = CollParams{reinterpret_cast<float *const *>(coll->peer_bufs), coll->rank, coll->world, coll->epoch,
                        coll->max_lanes};
  }
  dpo_loss_kernel<128, DpoParams><<<n_pairs, 128, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("aa_dpo_loss");
}

extern "C" int aa_dpo_loss_obj(const void *policy_lp, const void *ref_lp, int lp_dtype, int32_t n_pairs,
                               int32_t width, int64_t lp_row_stride, float scale_coeff, int mode, int loss_type,
                               float label_smoothing, float rpo_alpha, const int32_t *counts,
                               const int64_t *input_ids, int32_t L, int64_t ids_row_stride, float *per_pair,
                               float *grad_seg, float *stats, uint32_t *counter, const int32_t *status,
                               void *stream) {
  AA_REQUIRE(n_pairs > 0 && width >= 0, AA_ERR_ARG, "aa_dpo_loss_obj: bad sizes");
  AA_REQUIRE(policy_lp && per_pair && grad_seg && stats && counter, AA_ERR_ARG, "aa_dpo_loss_obj: null pointer");
  AA_REQUIRE(lp_dtype == AA_BF16 || lp_dtype == AA_F16 || lp_dtype == AA_F32, AA_ERR_DTYPE,
             "aa_dpo_loss_obj: bad dtype %d", lp_dtype);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "aa_dpo_loss_obj: bad mode %d", mode);
  AA_REQUIRE(loss_type >= AA_DPO_SIGMOID && loss_type <= AA_DPO_APO_DOWN, AA_ERR_ARG,
             "aa_dpo_loss_obj: bad objective: loss_type %d", loss_type);
  const bool smoothable = loss_type == AA_DPO_SIGMOID || loss_type == AA_DPO_ROBUST;
  AA_REQUIRE(label_smoothing >= 0.f && label_smoothing < 0.5f && (smoothable || label_smoothing == 0.f), AA_ERR_ARG,
             "aa_dpo_loss_obj: bad objective: label_smoothing %g with loss_type %d", label_smoothing, loss_type);
  AA_REQUIRE(rpo_alpha >= 0.f && isfinite(rpo_alpha), AA_ERR_ARG, "aa_dpo_loss_obj: bad objective: rpo_alpha %g",
             rpo_alpha);
  AA_REQUIRE((loss_type != AA_DPO_IPO && loss_type != AA_DPO_SPPO_HARD) || (scale_coeff > 0.f && isfinite(scale_coeff)),
             AA_ERR_ARG, "aa_dpo_loss_obj: bad objective: loss_type %d needs scale_coeff > 0, got %g", loss_type,
             scale_coeff);
  AA_REQUIRE(counts || (loss_type != AA_DPO_IPO && rpo_alpha == 0.f), AA_ERR_ARG,
             "aa_dpo_loss_obj: loss_type %d with rpo_alpha %g needs the row counts", loss_type, rpo_alpha);
  DpoObjParams p{{policy_lp, ref_lp, lp_dtype, n_pairs, width, lp_row_stride, scale_coeff,
                  mode == AA_MODE_FAITHFUL ? lp_dtype : AA_F32, input_ids, L, ids_row_stride, per_pair, grad_seg,
                  stats, counter, nullptr, CollParams{nullptr, 0, 1, 0u, 0u}, status},
                 loss_type, label_smoothing, rpo_alpha, counts};
  dpo_loss_kernel<128, DpoObjParams><<<n_pairs, 128, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("aa_dpo_loss_obj");
}

extern "C" int aa_dpo_loss_ext(const void *policy_lp, const void *ref_lp, int lp_dtype, int32_t n_pairs,
                               int32_t width, int64_t lp_row_stride, float scale_coeff, int mode, int loss_type,
                               float label_smoothing, float rpo_alpha, int f_divergence, float f_alpha_coef,
                               float discopop_tau, float exo_log_keep, float exo_log_smooth, const int32_t *counts, const int64_t *input_ids, int32_t L,
                               int64_t ids_row_stride, float *per_pair, float *grad_seg, float *stats,
                               uint32_t *counter, const int32_t *status, void *stream) {
  AA_REQUIRE(n_pairs > 0 && width >= 0, AA_ERR_ARG, "aa_dpo_loss_ext: bad sizes");
  AA_REQUIRE(policy_lp && per_pair && grad_seg && stats && counter, AA_ERR_ARG, "aa_dpo_loss_ext: null pointer");
  AA_REQUIRE(lp_dtype == AA_BF16 || lp_dtype == AA_F16 || lp_dtype == AA_F32, AA_ERR_DTYPE,
             "aa_dpo_loss_ext: bad dtype %d", lp_dtype);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "aa_dpo_loss_ext: bad mode %d", mode);
  AA_REQUIRE(loss_type >= AA_DPO_SIGMOID && loss_type <= AA_DPO_AOT_PAIR, AA_ERR_ARG,
             "aa_dpo_loss_ext: bad objective: loss_type %d", loss_type);
  AA_REQUIRE(f_divergence >= AA_DPO_FDIV_REVERSE_KL && f_divergence <= AA_DPO_FDIV_ALPHA, AA_ERR_ARG,
             "aa_dpo_loss_ext: bad objective: f_divergence %d", f_divergence);
  const bool smoothable = loss_type == AA_DPO_SIGMOID || loss_type == AA_DPO_ROBUST || loss_type == AA_DPO_EXO_PAIR ||
                          loss_type == AA_DPO_AOT || loss_type == AA_DPO_AOT_PAIR;
  AA_REQUIRE(label_smoothing >= 0.f && label_smoothing < 0.5f && (smoothable || label_smoothing == 0.f), AA_ERR_ARG,
             "aa_dpo_loss_ext: bad objective: label_smoothing %g with loss_type %d", label_smoothing, loss_type);
  AA_REQUIRE(rpo_alpha >= 0.f && isfinite(rpo_alpha), AA_ERR_ARG, "aa_dpo_loss_ext: bad objective: rpo_alpha %g",
             rpo_alpha);
  AA_REQUIRE((loss_type != AA_DPO_IPO && loss_type != AA_DPO_SPPO_HARD) || (scale_coeff > 0.f && isfinite(scale_coeff)),
             AA_ERR_ARG, "aa_dpo_loss_ext: bad objective: loss_type %d needs scale_coeff > 0, got %g", loss_type,
             scale_coeff);
  const bool reads_h = loss_type == AA_DPO_SIGMOID || loss_type == AA_DPO_ROBUST || loss_type == AA_DPO_HINGE ||
                       loss_type == AA_DPO_EXO_PAIR;
  AA_REQUIRE(f_divergence == AA_DPO_FDIV_REVERSE_KL || reads_h, AA_ERR_ARG,
             "aa_dpo_loss_ext: bad objective: f_divergence %d with loss_type %d", f_divergence, loss_type);
  AA_REQUIRE(f_alpha_coef > 0.f && isfinite(f_alpha_coef) && (f_alpha_coef == 1.f || f_divergence == AA_DPO_FDIV_ALPHA),
             AA_ERR_ARG, "aa_dpo_loss_ext: bad objective: f_alpha_coef %g with f_divergence %d", f_alpha_coef,
             f_divergence);
  AA_REQUIRE(discopop_tau > 0.f && isfinite(discopop_tau) && (discopop_tau == 0.05f || loss_type == AA_DPO_DISCOPOP),
             AA_ERR_ARG, "aa_dpo_loss_ext: bad objective: discopop_tau %g with loss_type %d", discopop_tau, loss_type);
  AA_REQUIRE(loss_type != AA_DPO_EXO_PAIR || (exo_log_keep < 0.f && exo_log_smooth < 0.f && isfinite(exo_log_smooth)),
             AA_ERR_ARG, "aa_dpo_loss_ext: bad objective: EXO's log(1 - e') %g and log(e') %g", exo_log_keep,
             exo_log_smooth);
  AA_REQUIRE((loss_type != AA_DPO_AOT && loss_type != AA_DPO_AOT_PAIR) || n_pairs <= AA_DPO_AOT_MAX_PAIRS, AA_ERR_ARG,
             "aa_dpo_loss_ext: AOT sorts at most %d pairs, got %d", AA_DPO_AOT_MAX_PAIRS, n_pairs);
  AA_REQUIRE(counts || (loss_type != AA_DPO_IPO && rpo_alpha == 0.f), AA_ERR_ARG,
             "aa_dpo_loss_ext: loss_type %d with rpo_alpha %g needs the row counts", loss_type, rpo_alpha);
  const double dt_max = lp_dtype == AA_F16 ? 65504.0 : lp_dtype == AA_BF16 ? 3.3895313892515355e38 : 3.4028234663852886e38;
  DpoExtParams p;
  static_cast<DpoObjParams &>(p) =
      DpoObjParams{{policy_lp, ref_lp, lp_dtype, n_pairs, width, lp_row_stride, scale_coeff,
                    mode == AA_MODE_FAITHFUL ? lp_dtype : AA_F32, input_ids, L, ids_row_stride, per_pair, grad_seg,
                    stats, counter, nullptr, CollParams{nullptr, 0, 1, 0u, 0u}, status},
                   loss_type, label_smoothing, rpo_alpha, counts};
  p.fdiv = f_divergence;
  p.f_alpha = f_alpha_coef;
  p.tau = discopop_tau;
  p.exp_cap = static_cast<float>(floor(log(dt_max) * 1e4) / 1e4);
  p.exo_c1 = exo_log_keep;
  p.exo_c2 = exo_log_smooth;
  dpo_loss_kernel<128, DpoExtParams><<<n_pairs, 128, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch("aa_dpo_loss_ext");
}
