// logprob_fused.cu -- K1f: log-probs, the loss's per-token gradient and the gradient tile in ONE pass over the logits tile,
// for losses that are (masked) means of per-token terms: the PPO actor loss (described below), the causal-LM cross-entropy
// (aa_logprob_ce_fused: trainers/text_to_text/sft.py:95-98, ppo.py:400-408) and the GRPO loss (aa_logprob_grpo_fused:
// trainers/text_to_text/grpo.py:290-312).  The three differ only in the record the prep kernel writes per row and in the
// per-token function the boundary thread calls (csrc/ppo_math.cuh).
//
// Reference: trainers/text_image_to_text/ppo.py:296-316 (text: trainers/text_to_text/ppo.py:336-349):
//     logits = actor(**batch).logits ; log_probs = gather_log_probabilities(logits[b, :-1][-R:], ids[b, 1:][-R:])
//     actor_loss = actor_loss_fn(log_probs, old_log_probs, advantages, mask) ; actor_model.backward(actor_loss)
// i.e. K1 (read the scored rows) -> K5 -> K1b (read the scored rows AGAIN, write the gradient tile).
//
// The clipped-ratio objective is a masked MEAN of per-token terms: d loss / d log_prob[b, t] depends on that token's own
// log-prob, on (old_log_prob, advantage, mask)[b, t] and on the row's mask count -- all known before the forward.  So
// the gradient row can be produced right after the row's (max, logsum), while the row is still on the chip:
//
//   per scored row, one CTA:   phase A  stream the row through a shared-memory ring (cp.async.bulk), online softmax
//                              boundary one thread: log-prob -> actor_token() -> g = d loss / d log-prob
//                              phase B  stream the SAME row again -- 304 KB at V = 152064, read a few microseconds ago
//                                       by this CTA, so the copy engine finds it in the 50 MB L2 (phase-A loads carry
//                                       an L2 evict_last policy, phase-B loads and the stores evict_first) --
//                                       g * (onehot - softmax) in place in shared memory, cp.async.bulk stores.
//
// HBM traffic per scored row: V*e read + V*e written instead of 2*V*e read + V*e written (K1 + K1b); unscored tile rows
// are written by the copy engine from a zeroed buffer, as in K1b.  The loss VALUE is still reduced by K5 from the
// log-probs this kernel writes (a 16 us launch); autograd's backward returns the tile produced here, multiplied in
// place by the incoming scalar only if that is not 1 (aa_scale_tile: every CTA reads the scalar and leaves).
#include <atomic>

#include "common.cuh"
#include "logprob_math.cuh"
#include "ppo_math.cuh"

namespace aa {

struct FusedActorParams {
  const void *logits;
  int64_t row_stride;
  int V;
  // PM kernels (aa_logprob_actor_fused_pm, aa_logprob_grpo_fused_pm): kinds 0 and 3 take CISPO or SAPO (pm, AA_PM_*)
  // with SAPO's temperatures tau_pos / tau_neg in place of the clipped ratio (ppo_math.cuh, pm_token / grpo_pm_token),
  // and rp is s's dtype.  The three fields sit in the struct's alignment holes, so that the parameter block keeps its
  // size and layout and the other kernels their code.
  int pm;
  const int64_t *labels;
  RowMap map;
  const int64_t *seg_tile_row;
  int seq;  // tile rows per segment (n_tile_rows / n_seg)
  void *out;
  int out_dtype;
  float tau_pos;  // PM
  float *stat_max, *stat_logsum;  // optional
  const void *old;
  int64_t old_stride;
  const void *adv;
  int64_t adv_stride;
  int adv_dtype;
  float tau_neg;  // PM
  const uint8_t *mask;
  int64_t mask_stride;
  int W;
  float clip;
  int rx, rp;
  // kind 0 objective (aa_logprob_actor_fused_obj; otherwise clip_hi = clip, dual = 0, agg = seq-mean-token-mean): clip
  // range [1 - clip, 1 + clip_hi], dual-clip factor (0 = off) with `dual * adv` rounded to ra, loss aggregation
  float clip_hi, dual;
  int ra, agg;
  void *grad;
  int64_t grad_row_stride;
  int32_t *status;
  float log2e, zero;
  int interleave;  // size of the persistent grid: the work list alternates `interleave` scored rows / zero rows
  // kind 1 (cross-entropy, aa_logprob_ce_fused): every row whose label != ignore_index has the SAME upstream gradient
  // *ce_coeff = -loss_scale / n_valid (written by ce_coeff_kernel); old / adv / mask are unused
  // kind 2 (GRPO, aa_logprob_grpo_fused): old = reference log-probs, adv = ONE fp32 advantage per segment, clip = beta,
  // a token counts while j < row_end[segment], 1 / *total is d loss / d per-token loss (grpo_mask_kernel wrote both)
  // kind 3 (GRPO's clipped objective, aa_logprob_grpo_fused_obj): kind 2's fields, W = K, the clip range
  // [1 - clip_lo, 1 + clip_hi], dual (0 = off) and agg (grpo_agg_coeff gives g_rs); old_pol: the rollout-time policy
  // log-probs at the log-prob's own index (out_idx), or nullptr for the pass's own log-probs (ratio 1)
  int kind;
  const void *old_pol;
  float clip_lo;
  int kl_est;  // kind 3: the per-token KL's estimator (AA_KL_*; aa_logprob_grpo_fused_obj: AA_KL_K3); kind 0: the KL term's
  int64_t ignore_index;
  const float *ce_coeff;
  const int32_t *row_end;
  const float *total;
  float *entropy;  // ENT kernels: fp32 entropy of every scored row at its log-prob's position (phase A)
  // EGRAD kernels (entropy bonus, loss - ent_coeff * mean entropy): the row's g_H = d loss / d H is
  // kind 0: ent_seg[segment] (= -ent_coeff / (n_seg * mask count), the masked mean's coefficient, or -ent_coeff / total
  // mask count under token-mean, written by the prep kernel) for masked-in tokens; kind 2: -ent_coeff * g_rs (= -ent_coeff / counted tokens) for counted tokens
  float ent_coeff;
  float *ent_seg;
  // kind 0 KL loss term (aa_logprob_actor_fused_kl; kl_coeff 0 = off): the KL of the token's log-prob against
  // ref[out_idx] (the reference log-probs laid out like `out`) by estimator kl_est adds its gradient to the token's;
  // kl_seg[segment] = d total / d KL of a masked-in token (kl_term_coeff, written by the prep kernel)
  const void *ref;
  float kl_coeff;
  float *kl_seg;
};

// One record per gradient-tile row, in the order the persistent kernel walks them.  The scored rows are bound by
// instruction issue / MUFU (two exp per logit in one kernel), the zero rows are pure copy-engine stores: the list
// alternates G scored rows and G zero rows (G = grid size), so every CTA's producer lane fires the stores of a zero
// row while its consumer warps are still busy with the scored row before it -- the zero rows ride in the DRAM
// bandwidth the compute-bound rows leave unused.
struct __align__(16) FusedRec {
  int64_t x_off;    // element offset of the logits row
  int64_t g_row;    // row index in the gradient tile
  int64_t out_idx;  // element index of the log-prob in `out` (and of old / adv / mask relative to their row starts)
  float old, adv, g_rs;
  int32_t y;        // label column; -1: out of range; -2: zero row
  int32_t flat;     // index into stat_max / stat_logsum
  int32_t on;       // mask bit
};
static_assert(sizeof(FusedRec) == 48, "FusedRec is read as three 16-byte vectors");
static_assert(sizeof(FusedActorParams) == 344, "the PM fields fill alignment holes: the parameter block keeps its size");

// grid (ceil(seq / 256), n_seg): block (c, seg) resolves tile rows [256 c, 256 c + 256) of sample `seg`.
template <bool EGRAD = false>
__global__ void __launch_bounds__(256) fused_actor_prep_kernel(const FusedActorParams p, FusedRec *__restrict__ rec) {
  __shared__ float scratch[33];
  const int seg = blockIdx.y, tid = threadIdx.x;
  const int k = blockIdx.x * 256 + tid;
  float cnt = 0.f;
  const bool token_mean = p.kind == 0 && p.agg == AA_AGG_TOKEN_MEAN;
  if (p.kind == 0) {
    // token-mean: the mask count of the whole micro-batch (every block counts it; no host sync, no extra launch)
    for (int k = token_mean ? 0 : seg; k < (token_mean ? p.map.n_seg : seg + 1); ++k)
      for (int t = tid; t < p.W; t += 256) cnt += p.mask[k * p.mask_stride + t] ? 1.f : 0.f;
    cnt = block_sum<256>(cnt, scratch);
    if constexpr (EGRAD) {
      if (blockIdx.x == 0 && tid == 0)
        p.ent_seg[seg] = -p.ent_coeff / (token_mean ? cnt : static_cast<float>(p.map.n_seg) * cnt);
    }
    if (p.kl_coeff != 0.f && blockIdx.x == 0 && tid == 0)
      p.kl_seg[seg] = kl_term_coeff(p.kl_coeff, p.agg, cnt, p.map.n_seg, p.rx);
  }
  if (k >= p.seq) return;
  const int64_t work = static_cast<int64_t>(seg) * p.seq + k;
  const int64_t first_flat = __ldg(p.map.seg_cum + seg);
  const int64_t n = __ldg(p.map.seg_cum + seg + 1) - first_flat;
  const int64_t total = __ldg(p.map.seg_cum + p.map.n_seg);
  const int64_t j = work - __ldg(p.seg_tile_row + seg);
  const bool scored = j >= 0 && j < n;
  const int64_t scored_before = first_flat + min(max(j, static_cast<int64_t>(0)), n);
  const int64_t G = p.interleave, Z = static_cast<int64_t>(p.map.n_seg) * p.seq - total;
  int64_t slot;
  if (scored) {
    const int64_t i = first_flat + j;
    slot = i + min((i / G) * G, Z);                // zero rows of the earlier rounds come first
  } else {
    const int64_t z = work - scored_before;
    slot = min((z / G + 1) * G, total) + z;        // scored rows of this and the earlier rounds come first
  }
  FusedRec r;
  r.x_off = 0; r.g_row = work; r.out_idx = 0; r.old = 0.f; r.adv = 0.f; r.g_rs = 0.f; r.y = -2; r.flat = 0; r.on = 0;
  if (scored) {
    const int64_t y = __ldg(p.labels + __ldg(p.map.seg_label_off + seg) + j);
    if (p.kind != 1 || y != p.ignore_index) {  // cross-entropy: an ignored position is a zero row (its log-prob stays 0: no traffic)
      r.x_off = __ldg(p.map.seg_logit_off + seg) + j * p.row_stride;
      r.out_idx = __ldg(p.map.seg_out_off + seg) + j;
      r.y = (y >= 0 && y < p.V) ? static_cast<int32_t>(y) : -1;
      r.flat = static_cast<int32_t>(first_flat + j);
      if (p.kind == 0) {
        r.old = load_as_float(p.old, seg * p.old_stride + j, p.out_dtype);
        r.adv = load_as_float(p.adv, seg * p.adv_stride + j, p.adv_dtype);
        r.g_rs = token_mean ? actor_token_mean_coeff(cnt, p.rp) : actor_row_coeff(cnt, p.map.n_seg, p.rp);
        r.on = p.mask[seg * p.mask_stride + j] ? 1 : 0;
      } else if (p.kind >= 2) {
        const int end = __ldg(p.row_end + seg);
        r.old = load_as_float(p.old, seg * p.old_stride + j, p.out_dtype);
        r.adv = reinterpret_cast<const float *>(p.adv)[seg];
        r.g_rs = (p.kind == 2) ? 1.f / __ldg(p.total)
                               : grpo_agg_coeff(p.agg, __ldg(p.total), static_cast<float>(end), p.map.n_seg, p.W);
        r.on = (j < end) ? 1 : 0;
      } else {
        r.g_rs = __ldg(p.ce_coeff);
        r.on = 1;
      }
    }
  }
  rec[slot] = r;
}

namespace bulk {
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void bulk_g2s_hint(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar,
                                              uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
}
__device__ __forceinline__ void bulk_s2g_hint(void *dst_gmem, const void *src_smem, uint32_t bytes, uint64_t pol) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(dst_gmem),
               "r"(smem_u32(src_smem)), "r"(bytes), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
}  // namespace bulk

// vec_grad (logprob_math.cuh) with the reference's 16-bit rounding of the log-softmax done by ONE F2FP.PACK_AB per pair
// (+ two ALU unpacks) instead of the Veltkamp split on the FMA pipe (FFMA2 + 2 FADD2): the same bits for finite values,
// -inf logits need no clamp (HMNMX2), and three instructions per pair move from the FMA-heavy pipe -- the busiest one
// of this kernel, 57 % -- to the ALU pipe (36 %).  K1b keeps the split: it is HBM-bound with the XU pipe as runner-up.
template <typename T, bool FAITHFUL>
__device__ __forceinline__ uint4 vec_grad_pk(const uint4 &v, const GradConsts &k) {
  if constexpr (sizeof(T) == 4 || !FAITHFUL) {
    return vec_grad<T, FAITHFUL>(v, k);
  } else {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float lo, hi;
      unpack2<T>(w[i], lo, hi);
      f2_unpack(f2_sub(f2_sub(f2_pack(lo, hi), k.m2), k.ls2), lo, hi);
      unpack2<T>(pack2<T>(lo, hi), lo, hi);  // round_T((x - max) - logsum): what ATen's backward re-reads
      f2_unpack(f2_mul(f2_ex2(f2_mul(f2_pack(lo, hi), f2_splat(kLog2e))), k.ng2), lo, hi);
      o[i] = pack2<T>(lo, hi);
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// EGRAD (implies ENT): phase B adds the entropy's gradient (logprob_math.cuh, vec_grad_ent) to rows with g_H != 0.
// PM: kinds 0 and 3 run the policy loss p.pm (CISPO / SAPO) at the boundary; a flag of its own, so that the other
// instantiations keep their code.
template <typename T, int CONSUMERS, int STAGES, int UNROLL, int LAG, bool FAITHFUL, bool ENT = false, bool EGRAD = false,
          bool PM = false>
__global__ void __launch_bounds__(CONSUMERS + 32)
    logprob_actor_fused_kernel(const FusedActorParams p, const FusedRec *__restrict__ rec, int64_t n_work) {
  constexpr int E = Traits<T>::kVec;
  constexpr int STAGE_VECS = CONSUMERS * UNROLL;
  constexpr int NW = CONSUMERS / kWarp;
  static_assert(LAG >= 2 && LAG < STAGES, "phase A holds two stages at a time; LAG must leave at least one free stage");
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint4 *ring = reinterpret_cast<uint4 *>(smem_raw);
  uint4 *zero_buf = ring + static_cast<size_t>(STAGES) * STAGE_VECS;
  uint64_t *full = reinterpret_cast<uint64_t *>(zero_buf + STAGE_VECS);
  uint64_t *done = full + STAGES;
  uint64_t *st_dst = done + STAGES;  // destination of the chunk held by each stage (phase B), 0 for phase A
  uint32_t *st_bytes = reinterpret_cast<uint32_t *>(st_dst + STAGES);
  static_assert(ENT || !EGRAD, "the entropy gradient needs the entropy");
  __shared__ float sh_m[32], sh_s[32], sh_b[EGRAD ? 8 : 4];
  __shared__ float sh_t[ENT ? 32 : 1];
  const int tid = threadIdx.x;
  const int V = p.V;
  const T *__restrict__ logits = reinterpret_cast<const T *>(p.logits);
  T *__restrict__ grad = reinterpret_cast<T *>(p.grad);
  for (int i = tid; i < STAGE_VECS; i += CONSUMERS + 32) zero_buf[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) {
      bulk::mbar_init(full + i, 1);
      bulk::mbar_init(done + i, NW);
    }
    bulk::fence_barrier_init();
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // zero_buf is read by the async proxy
  __syncthreads();

  if (tid >= CONSUMERS) {
    // ------------------------------ producer lane ------------------------------
    if (tid != CONSUMERS) return;
    const uint64_t pol_keep = bulk::policy_evict_last(), pol_drop = bulk::policy_evict_first();
    // ring positions are kept as (stage, parity) pairs stepped by hand: `it % STAGES` with a 64-bit counter and
    // STAGES = 6 is a ~40-instruction division per chunk (seen in the SASS of the first version)
    int inflight = 0;                     // chunks loaded and not yet handed back
    int ld_stage = 0;                     // stage of the next load
    int rt_stage = 0;                     // stage of the next chunk to hand back (phase A: freed; phase B: stored)
    uint32_t rt_phase = 0;
    auto retire_one = [&]() {
      const int s = rt_stage;
      bulk::mbar_wait(done + s, rt_phase);
      if (st_bytes[s])
        bulk::bulk_s2g_hint(reinterpret_cast<void *>(st_dst[s]), ring + static_cast<size_t>(s) * STAGE_VECS, st_bytes[s],
                            pol_drop);
      bulk::commit_group();  // one (possibly empty) group per chunk: wait_group.read below counts chunks
      --inflight;
      if (++rt_stage == STAGES) {
        rt_stage = 0;
        rt_phase ^= 1u;
      }
    };
    // zero rows are not stored in one burst: their chunks are fed to the copy engine one per chunk load of the scored
    // row that follows, so the engine's queue never holds a whole 300 KB row in front of the loads the consumers wait for
    uint4 *zq_dst = nullptr;
    int zq_left = 0;  // vectors of the pending zero row not yet handed to the copy engine
    auto zero_some = [&](int max_chunks) {
      while (zq_left > 0 && max_chunks-- > 0) {
        const int n = min(STAGE_VECS, zq_left);
        bulk::bulk_s2g_hint(zq_dst, zero_buf, static_cast<uint32_t>(n) * 16u, pol_drop);
        zq_dst += n;
        zq_left -= n;
      }
    };
    for (int64_t r = blockIdx.x; r < n_work; r += gridDim.x) {
      const int4 r0 = __ldg(reinterpret_cast<const int4 *>(rec + r));
      const int4 r2 = __ldg(reinterpret_cast<const int4 *>(rec + r) + 2);
      const int64_t x_off = (static_cast<int64_t>(static_cast<uint32_t>(r0.y)) << 32) | static_cast<uint32_t>(r0.x);
      const int64_t g_row = (static_cast<int64_t>(static_cast<uint32_t>(r0.w)) << 32) | static_cast<uint32_t>(r0.z);
      const int y = r2.y, on = r2.w;
      T *g_out = grad + g_row * p.grad_row_stride;
      const T *x = logits + x_off;
      const bool same_phase = ((reinterpret_cast<uintptr_t>(x) ^ reinterpret_cast<uintptr_t>(g_out)) & 15) == 0;
      // geometry of the row the chunks come from (scored rows: the logits row; it shares g_out's 16-byte phase)
      const uintptr_t ref = (y == -2) ? reinterpret_cast<uintptr_t>(g_out) : reinterpret_cast<uintptr_t>(x);
      const int mis = static_cast<int>((ref & 15) / sizeof(T));
      const int head = mis ? min(E - mis, V) : 0;
      const int nvec = (V - head) / E;
      const int tail0 = head + nvec * E;
      const uint4 *xbody = reinterpret_cast<const uint4 *>(x + head);
      uint4 *gbody = reinterpret_cast<uint4 *>(g_out + head);
      if (y != -2 && same_phase) {
        for (int ph = 0; ph < (on ? 2 : 1); ++ph) {
          for (int v0 = 0; v0 < nvec; v0 += STAGE_VECS) {
            const uint32_t bytes = static_cast<uint32_t>(min(STAGE_VECS, nvec - v0)) * 16u;
            while (inflight >= LAG) retire_one();
            const int s = ld_stage;
            // the stage's previous chunk was handed to the copy engine at least STAGES - LAG groups ago: wait until the
            // engine has finished READING it (later groups may stay pending)
            asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(STAGES - LAG) : "memory");
            st_dst[s] = reinterpret_cast<uint64_t>(gbody + v0);
            st_bytes[s] = ph ? bytes : 0u;
            bulk::mbar_expect_tx(full + s, bytes);
            bulk::bulk_g2s_hint(ring + static_cast<size_t>(s) * STAGE_VECS, xbody + v0, bytes, full + s,
                                ph ? pol_drop : pol_keep);
            ++inflight;
            if (++ld_stage == STAGES) ld_stage = 0;
            zero_some(1);  // joins the group of the next retired chunk
          }
        }
      }
      if (y == -2 || (!on && same_phase)) {  // zero row: the copy engine writes it from the zero buffer
        zero_some(1 << 30);                  // (whatever is left of the previous one first)
        for (int e = 0; e < head; ++e) g_out[e] = Traits<T>::from_float(0.f);
        for (int e = tail0; e < V; ++e) g_out[e] = Traits<T>::from_float(0.f);
        zq_dst = gbody;
        zq_left = nvec;
      }
    }
    zero_some(1 << 30);
    bulk::commit_group();
    while (inflight > 0) retire_one();
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // smem must outlive the engine's reads / the stores
    return;
  }

  // ------------------------------ consumer warps ------------------------------
  const f32x2 L2 = f2_splat(p.log2e);
  const int lane = tid & 31, wid = tid >> 5;
  int stage = 0;       // ring position of the next chunk, stepped by hand (see the producer)
  uint32_t phase = 0;
  for (int64_t r = blockIdx.x; r < n_work; r += gridDim.x) {
    const int4 r0 = __ldg(reinterpret_cast<const int4 *>(rec + r));
    const int4 r1 = __ldg(reinterpret_cast<const int4 *>(rec + r) + 1);
    const int4 r2 = __ldg(reinterpret_cast<const int4 *>(rec + r) + 2);
    const int y = r2.y;
    if (y == -2) continue;
    const int64_t x_off = (static_cast<int64_t>(static_cast<uint32_t>(r0.y)) << 32) | static_cast<uint32_t>(r0.x);
    const int64_t g_row = (static_cast<int64_t>(static_cast<uint32_t>(r0.w)) << 32) | static_cast<uint32_t>(r0.z);
    const int64_t out_idx = (static_cast<int64_t>(static_cast<uint32_t>(r1.y)) << 32) | static_cast<uint32_t>(r1.x);
    const float old = __int_as_float(r1.z), adv = __int_as_float(r1.w), g_rs = __int_as_float(r2.x);
    const int flat = r2.z;
    const bool on = r2.w != 0;
    T *g_out = grad + g_row * p.grad_row_stride;
    const T *x = logits + x_off;
    const bool same_phase = ((reinterpret_cast<uintptr_t>(x) ^ reinterpret_cast<uintptr_t>(g_out)) & 15) == 0;
    const int mis = static_cast<int>((reinterpret_cast<uintptr_t>(x) & 15) / sizeof(T));
    const int head = mis ? min(E - mis, V) : 0;
    const int nvec = (V - head) / E;
    const int tail0 = head + nvec * E;

    float xy = 0.f;
    if (tid == 0) xy = (y >= 0) ? Traits<T>::to_float(x[y]) : NAN;  // label column, issued before the streaming loop

    // ---- phase A: (max, sum exp) of the row ----
    float m = -INFINITY, s = 0.f, t = 0.f;
    if (same_phase) {
      if (tid < head) lse_push_t<ENT>(m, s, t, Traits<T>::to_float(x[tid]));
      if (tid < V - tail0) lse_push_t<ENT>(m, s, t, Traits<T>::to_float(x[tail0 + tid]));
      // two stages per fold: the running-max rescale (one MUFU, a compare and a select) is paid per 4 vectors
      for (int v0 = 0; v0 < nvec; v0 += 2 * STAGE_VECS) {
        const int n0 = min(STAGE_VECS, nvec - v0);
        const int n1 = min(STAGE_VECS, max(nvec - v0 - STAGE_VECS, 0));  // 0: the row ends in the first stage
        const int st0 = stage;
        const uint32_t ph0 = phase;
        int st1 = st0 + 1;
        uint32_t ph1 = ph0;
        if (st1 == STAGES) {
          st1 = 0;
          ph1 ^= 1u;
        }
        uint4 v[2 * UNROLL];
        bulk::mbar_wait(full + st0, ph0);
        const uint4 *buf0 = ring + static_cast<size_t>(st0) * STAGE_VECS;
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
          const int k = tid + u * CONSUMERS;
          v[u] = (k < n0) ? buf0[k] : bulk::neg_inf_vec<T>();
        }
        if (n1 > 0) {
          bulk::mbar_wait(full + st1, ph1);
          const uint4 *buf1 = ring + static_cast<size_t>(st1) * STAGE_VECS;
#pragma unroll
          for (int u = 0; u < UNROLL; ++u) {
            const int k = tid + u * CONSUMERS;
            v[UNROLL + u] = (k < n1) ? buf1[k] : bulk::neg_inf_vec<T>();
          }
        } else {
#pragma unroll
          for (int u = 0; u < UNROLL; ++u) v[UNROLL + u] = bulk::neg_inf_vec<T>();
        }
        // order this warp's generic-proxy reads of the stages before the copy engine's next write to them
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) {
          bulk::mbar_arrive(done + st0);
          if (n1 > 0) bulk::mbar_arrive(done + st1);
        }
        fold_batch_t<T, 2 * UNROLL, ENT>(v, m, s, t, L2);
        stage = st1;
        phase = ph1;
        if (n1 > 0 && ++stage == STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }
    } else {  // logits view and gradient tile disagree on the 16-byte phase of this row: element loops, no staging
      for (int e = tid; e < V; e += CONSUMERS) lse_push_t<ENT>(m, s, t, Traits<T>::to_float(x[e]));
    }
    // merge the partials of the CONSUMERS threads (named barrier 1: the producer warp is not part of it)
    warp_lse_t<ENT>(m, s, t);
    if (lane == 0) {
      sh_m[wid] = m;
      sh_s[wid] = s;
      if constexpr (ENT) sh_t[wid] = t;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
    if (wid == 0) {
      m = lane < NW ? sh_m[lane] : -INFINITY;
      s = lane < NW ? sh_s[lane] : 0.f;
      if constexpr (ENT) t = lane < NW ? sh_t[lane] : 0.f;
      warp_lse_t<ENT>(m, s, t);
      if (lane == 0) {
        // ---- boundary: log-prob -> d loss / d log-prob of this token ----
        const float logsum = logf(s);
        float lp = (xy - m) - logsum;  // same association as ATen's `x - max - log(sum)`
        if (y < 0) {
          lp = NAN;
          if (p.status) atomicOr(p.status, AA_STATUS_LABEL_OOB);
        }
        store_from_float(p.out, out_idx, p.out_dtype, lp);
        if constexpr (ENT) p.entropy[out_idx] = entropy_of(logsum, s, t);
        if (p.stat_max) {
          p.stat_max[flat] = m;
          p.stat_logsum[flat] = logsum;
        }
        float obj, g = g_rs;  // cross-entropy: the same -loss_scale / n_valid for every scored row
        int why;
        if (p.kind == 0) {
          const float lpr = round_to(lp, p.out_dtype);
          if constexpr (PM)
            pm_token(p.pm, lpr, old, adv, on, g_rs, p.clip_hi, p.tau_pos, p.tau_neg, p.rx, p.rp, obj, g, why);
          else
            actor_token(lpr, old, adv, on, g_rs, p.clip, p.clip_hi, p.dual, p.rx, p.rp, p.ra, obj, g, why);
          if (p.kl_coeff != 0.f && on) {  // the KL term: its gradient is added after the ratio's (as in K5)
            float kaux;
            kl_value(lpr, load_as_float(p.ref, out_idx, p.out_dtype), p.kl_est, p.rx, kaux);
            g = kl_grad(g, __ldg(p.kl_seg + g_row / p.seq), p.kl_est, kaux, p.rx);
          }
        }
        if (p.kind == 2) grpo_token(round_to(lp, p.out_dtype), old, adv, on, g_rs, p.clip, p.rx, obj, g);
        if (p.kind == 3) {
          const float lpr = round_to(lp, p.out_dtype);
          const float po = p.old_pol ? load_as_float(p.old_pol, out_idx, p.out_dtype) : lpr;
          if constexpr (PM)
            grpo_pm_token(p.pm, lpr, po, old, adv, on, g_rs, p.clip, p.clip_hi, p.tau_pos, p.tau_neg, p.kl_est, p.rx,
                          obj, g, why);
          else
            grpo_obj_token(lpr, po, old, adv, on, g_rs, p.clip, p.clip_lo, p.clip_hi, p.dual, p.kl_est, p.rx, obj, g,
                           why);
        }
        sh_b[0] = m;
        sh_b[1] = logsum;
        sh_b[2] = g;
        if constexpr (EGRAD) {
          float gH = 0.f;
          // GRPO: a token mean over the completion mask under every aggregation (kind 3's g_rs is the loss's)
          if (on)
            gH = (p.kind == 0) ? __ldg(p.ent_seg + g_row / p.seq)
                               : -p.ent_coeff * ((p.kind == 2) ? g_rs : 1.f / __ldg(p.total));
          sh_b[3] = entropy_of(logsum, s, t);
          sh_b[4] = gH;
        }
      }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
    if (!on) {  // the producer zero-fills the row (same_phase) ...
      if (!same_phase)
        for (int e = tid; e < V; e += CONSUMERS) g_out[e] = Traits<T>::from_float(0.f);
      continue;
    }
    m = sh_b[0];
    const float logsum = sh_b[1], g = sh_b[2];
    float H = 0.f, gH = 0.f;
    if constexpr (EGRAD) {
      H = sh_b[3];
      gH = sh_b[4];
    }
    const bool ent = EGRAD && gH != 0.f;  // rows without an entropy gradient run the plain code

    // ---- phase B: g * (onehot - softmax), the row comes from L2 ----
    const float lse = m + logsum;
    const float c_f32 = -lse * kLog2e;
    const float neg_g = FAITHFUL ? -g : -g * ex2_approx(fmaf(-lse, kLog2e, -c_f32));
    const GradConsts gk = make_grad_consts(m, logsum, c_f32, neg_g, p.zero);
    const float ngh = !EGRAD ? 0.f : FAITHFUL ? -gH : -gH * ex2_approx(fmaf(-lse, kLog2e, -c_f32));
    const EntConsts ek{f2_splat(H), f2_splat(ngh)};
    const bool dead = (g == 0.f) && !ent;  // clipped token: 0 * softmax, written as +0 like K1b's zero rows
#define AA_K1F_ELEM(c)                                                                                        \
  (EGRAD ? grad_of_ent<T, FAITHFUL>(Traits<T>::to_float(x[c]), m, logsum, c_f32, neg_g, g, (c) == y, ent, ngh, H) \
         : grad_of<T, FAITHFUL>(Traits<T>::to_float(x[c]), m, logsum, c_f32, neg_g, g, (c) == y))
    if (!same_phase) {
      for (int e = tid; e < V; e += CONSUMERS) g_out[e] = Traits<T>::from_float(dead ? 0.f : AA_K1F_ELEM(e));
      continue;
    }
    if (tid < head) g_out[tid] = Traits<T>::from_float(dead ? 0.f : AA_K1F_ELEM(tid));
    if (tid < V - tail0) g_out[tail0 + tid] = Traits<T>::from_float(dead ? 0.f : AA_K1F_ELEM(tail0 + tid));
#undef AA_K1F_ELEM
    const int yv = (y >= head && y < tail0) ? (y - head) / E : -1;  // body vector holding the label column
    for (int v0 = 0; v0 < nvec; v0 += STAGE_VECS) {
      const int n = min(STAGE_VECS, nvec - v0);
      const int st = stage;
      bulk::mbar_wait(full + st, phase);
      uint4 *buf = ring + static_cast<size_t>(st) * STAGE_VECS;
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const int k = tid + u * CONSUMERS;
        if (k < n) {
          if (dead) {
            buf[k] = make_uint4(0, 0, 0, 0);
          } else {
            const uint4 in = buf[k];
            uint4 o = ent ? vec_grad_ent<T, FAITHFUL, true>(in, gk, ek) : vec_grad_pk<T, FAITHFUL>(in, gk);
            if (v0 + k == yv)
              patch_label<T, FAITHFUL, EGRAD>(o, in, (y - head) - (v0 + k) * E, m, logsum, c_f32, neg_g, g, ent, ngh, H);
            buf[k] = o;
          }
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the copy engine
      __syncwarp();
      if (lane == 0) bulk::mbar_arrive(done + st);
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1u;
      }
    }
  }
}

// coeff[0] = -loss_scale / #(labels != ignore_index): the upstream gradient of every scored row of a mean cross-entropy
__global__ void __launch_bounds__(1024) ce_coeff_kernel(const int64_t *__restrict__ labels, int64_t n, int64_t ignore_index,
                                                        float loss_scale, float *__restrict__ coeff) {
  __shared__ float scratch[33];
  float c = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += 1024) c += (__ldg(labels + i) != ignore_index) ? 1.f : 0.f;
  c = block_sum<1024>(c, scratch);
  if (threadIdx.x == 0) coeff[0] = -loss_scale / c;
}

// tile *= scale unless scale == 1 (every thread reads the scalar first: the usual case costs one empty launch)
template <typename T>
__global__ void __launch_bounds__(256) scale_tile_kernel(T *__restrict__ tile, int64_t n, const void *scale, int scale_dtype) {
  const float s = load_as_float(scale, 0, scale_dtype);
  if (s == 1.f) return;
  constexpr int E = Traits<T>::kVec;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const int64_t t0 = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int mis = static_cast<int>((reinterpret_cast<uintptr_t>(tile) & 15) / sizeof(T));
  const int64_t head = mis ? min(static_cast<int64_t>(E - mis), n) : 0;
  const int64_t nvec = (n - head) / E;
  const int64_t tail0 = head + nvec * E;
  if (t0 < head) tile[t0] = Traits<T>::from_float(Traits<T>::to_float(tile[t0]) * s);
  if (t0 < n - tail0) tile[tail0 + t0] = Traits<T>::from_float(Traits<T>::to_float(tile[tail0 + t0]) * s);
  uint4 *body = reinterpret_cast<uint4 *>(tile + head);
  for (int64_t k = t0; k < nvec; k += stride) {
    uint4 v = body[k];
    if constexpr (sizeof(T) == 4) {
      v.x = __float_as_uint(__uint_as_float(v.x) * s);
      v.y = __float_as_uint(__uint_as_float(v.y) * s);
      v.z = __float_as_uint(__uint_as_float(v.z) * s);
      v.w = __float_as_uint(__uint_as_float(v.w) * s);
    } else {
      uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float lo, hi;
        unpack2<T>(w[i], lo, hi);
        w[i] = pack2<T>(lo * s, hi * s);
      }
      v = make_uint4(w[0], w[1], w[2], w[3]);
    }
    body[k] = v;
  }
}

// ---- host side ----------------------------------------------------------------------------
// One launch shape: 992 consumers (31 warps + the producer warp = 1024 threads), 6 x 31 KB stages, lag 4, 1 CTA/SM, zero
// rows interleaved with the scored rows.  One CTA per SM keeps 132 rows (40 MB of 152064-token bf16 rows) between the
// two passes, inside the 50 MB L2, so the second pass is an L2 hit; with two rows in flight per SM part of it misses.
// The kernel is bound by the MUFU / conversion pipe and instruction issue (two exp per logit + the bf16 pack) rather
// than by HBM.
template <typename T, bool ENT = false, bool EGRAD = false, bool PM = false>
static int launch_fused_kernel(const FusedActorParams &p, int mode, FusedRec *rec, int64_t n_work, cudaStream_t st) {
  constexpr int CONSUMERS = 992, STAGES = 6, UNROLL = 2, LAG = 4;
  constexpr size_t smem = static_cast<size_t>(STAGES + 1) * CONSUMERS * UNROLL * 16 + STAGES * (8 + 8 + 8 + 4) + 16;
  const bool faithful = (mode == AA_MODE_FAITHFUL) && sizeof(T) == 2;
  auto kf = logprob_actor_fused_kernel<T, CONSUMERS, STAGES, UNROLL, LAG, true, ENT, EGRAD, PM>;
  auto kn = logprob_actor_fused_kernel<T, CONSUMERS, STAGES, UNROLL, LAG, false, ENT, EGRAD, PM>;
  static std::atomic<bool> configured{false};  // the attribute is idempotent: a race sets it twice, harmlessly
  if (!configured.load(std::memory_order_relaxed)) {
    cudaError_t e = cudaFuncSetAttribute(kf, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(kn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) {
      set_error("aa_logprob_actor_fused: cannot reserve %zu B of shared memory: %s", smem, cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    configured.store(true, std::memory_order_relaxed);
  }
  int64_t grid = sm_count();
  if (grid > n_work) grid = n_work;
  FusedActorParams q = p;
  q.interleave = static_cast<int>(grid);
  const dim3 pgrid((q.seq + 255) / 256, q.map.n_seg);
  fused_actor_prep_kernel<EGRAD><<<pgrid, 256, 0, st>>>(q, rec);
  int rc = check_launch("aa_logprob_actor_fused(prep)");
  if (rc) return rc;
  if (faithful)
    kf<<<static_cast<unsigned>(grid), CONSUMERS + 32, smem, st>>>(q, rec, n_work);
  else
    kn<<<static_cast<unsigned>(grid), CONSUMERS + 32, smem, st>>>(q, rec, n_work);
  return check_launch("aa_logprob_actor_fused");
}

// egrad: the entropy-bonus kernels (p.entropy set)
template <bool PM>
static int launch_fused_of(const FusedActorParams &p, int logits_dtype, int mode, FusedRec *rec, int64_t n_work,
                           cudaStream_t st, bool egrad) {
  if (egrad) {
    switch (logits_dtype) {
      case AA_BF16: return launch_fused_kernel<__nv_bfloat16, true, true, PM>(p, mode, rec, n_work, st);
      case AA_F16: return launch_fused_kernel<__half, true, true, PM>(p, mode, rec, n_work, st);
      case AA_F32: return launch_fused_kernel<float, true, true, PM>(p, mode, rec, n_work, st);
    }
    return AA_ERR_DTYPE;
  }
  if (p.entropy) {
    switch (logits_dtype) {
      case AA_BF16: return launch_fused_kernel<__nv_bfloat16, true, false, PM>(p, mode, rec, n_work, st);
      case AA_F16: return launch_fused_kernel<__half, true, false, PM>(p, mode, rec, n_work, st);
      case AA_F32: return launch_fused_kernel<float, true, false, PM>(p, mode, rec, n_work, st);
    }
    return AA_ERR_DTYPE;
  }
  switch (logits_dtype) {
    case AA_BF16: return launch_fused_kernel<__nv_bfloat16, false, false, PM>(p, mode, rec, n_work, st);
    case AA_F16: return launch_fused_kernel<__half, false, false, PM>(p, mode, rec, n_work, st);
    case AA_F32: return launch_fused_kernel<float, false, false, PM>(p, mode, rec, n_work, st);
  }
  return AA_ERR_DTYPE;
}

// p.pm != 0: the PM kernels
static int launch_fused(const FusedActorParams &p, int logits_dtype, int mode, FusedRec *rec, int64_t n_work,
                        cudaStream_t st, bool egrad = false) {
  return p.pm ? launch_fused_of<true>(p, logits_dtype, mode, rec, n_work, st, egrad)
              : launch_fused_of<false>(p, logits_dtype, mode, rec, n_work, st, egrad);
}

// The fields every kind sets; each entry point adds its own and the kind.
static FusedActorParams fused_params(const void *logits, int64_t row_stride, int32_t V, const int64_t *labels,
                                     int32_t n_segments, const int64_t *seg_logit_off, const int64_t *seg_label_off,
                                     const int64_t *seg_out_off, const int64_t *seg_cum, const int64_t *seg_tile_row,
                                     int64_t n_tile_rows, void *log_probs, int lp_dtype, void *grad_logits,
                                     int64_t grad_row_stride, int32_t *status) {
  FusedActorParams p{};
  p.logits = logits;
  p.row_stride = row_stride;
  p.V = V;
  p.labels = labels;
  p.map = RowMap{seg_logit_off, seg_label_off, seg_out_off, seg_cum, n_segments};
  p.seg_tile_row = seg_tile_row;
  p.seq = static_cast<int>(n_tile_rows / n_segments);
  p.out = log_probs;
  p.out_dtype = lp_dtype;
  p.grad = grad_logits;
  p.grad_row_stride = grad_row_stride;
  p.status = status;
  p.log2e = kLog2e;
  p.zero = 0.0f;
  return p;
}

static inline bool fdtype_ok(int dt) { return dt == AA_BF16 || dt == AA_F16 || dt == AA_F32; }
static inline int promote_dt(int a, int b) { return (a == b) ? a : AA_F32; }

}  // namespace aa

using namespace aa;

// the KL loss term of aa_logprob_actor_fused_kl
struct ActorKlTerm {
  const void *ref;
  float coeff;
  int est;
};

// the policy loss of the PM entry points (AA_PM_*) and SAPO's temperatures
struct PolicyLoss {
  int mode;
  float tau_pos, tau_neg;
};

// aa_logprob_actor_fused{,_entropy,_obj,_kl}: entropy == nullptr runs the plain kernels; kl == nullptr: no KL term
static int logprob_actor_fused(const char *who, float *entropy, float entropy_coeff, const void *logits, int logits_dtype,
                               int64_t row_stride, int32_t V, const int64_t *labels, int32_t n_segments,
                               const int64_t *seg_logit_off, const int64_t *seg_label_off, const int64_t *seg_out_off,
                               const int64_t *seg_cum, const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs,
                               int lp_dtype, float *stat_max, float *stat_logsum, const void *old_log_probs,
                               int64_t old_stride, const void *advantages, int64_t adv_stride, int adv_dtype,
                               const uint8_t *mask, int64_t mask_stride, int32_t W, float clip_low, float clip_high,
                               float dual_clip, int loss_agg, int mode, void *grad_logits, int64_t grad_row_stride,
                               void *row_scratch, int32_t *status, void *stream, const ActorKlTerm *kl = nullptr,
                               const PolicyLoss *pm = nullptr) {
  AA_REQUIRE(V > 0 && n_segments > 0 && W > 0 && n_tile_rows > 0 && n_tile_rows % n_segments == 0, AA_ERR_ARG,
             "%s: bad sizes (the gradient tile holds n_tile_rows / n_segments rows per sample)", who);
  AA_REQUIRE(logits && labels && seg_logit_off && seg_label_off && seg_out_off && seg_cum && seg_tile_row && log_probs &&
                 old_log_probs && advantages && mask && grad_logits && row_scratch,
             AA_ERR_ARG, "%s: null pointer", who);
  AA_REQUIRE((stat_max == nullptr) == (stat_logsum == nullptr), AA_ERR_ARG,
             "%s: stat_max and stat_logsum go together", who);
  AA_REQUIRE(fdtype_ok(logits_dtype) && fdtype_ok(lp_dtype) && fdtype_ok(adv_dtype), AA_ERR_DTYPE,
             "%s: bad dtype", who);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "%s: bad mode", who);
  AA_REQUIRE((reinterpret_cast<uintptr_t>(row_scratch) & 15) == 0, AA_ERR_ALIGN,
             "%s: row_scratch must be 16-byte aligned", who);
  AA_REQUIRE(n_tile_rows / n_segments < (1ll << 31) && n_tile_rows < (1ll << 31), AA_ERR_ARG,
             "%s: tile too large", who);
  const bool f = (mode == AA_MODE_FAITHFUL);
  FusedActorParams p = fused_params(logits, row_stride, V, labels, n_segments, seg_logit_off, seg_label_off, seg_out_off,
                                    seg_cum, seg_tile_row, n_tile_rows, log_probs, lp_dtype, grad_logits,
                                    grad_row_stride, status);
  p.kind = 0;
  p.stat_max = stat_max;
  p.stat_logsum = stat_logsum;
  p.old = old_log_probs;
  p.old_stride = old_stride;
  p.adv = advantages;
  p.adv_stride = adv_stride;
  p.adv_dtype = adv_dtype;
  p.mask = mask;
  p.mask_stride = mask_stride;
  p.W = W;
  p.clip = clip_low;
  p.clip_hi = clip_high;
  p.dual = dual_clip;
  p.agg = loss_agg;
  p.rx = f ? lp_dtype : AA_F32;
  p.rp = f ? promote_dt(lp_dtype, adv_dtype) : AA_F32;
  p.ra = f ? adv_dtype : AA_F32;
  if (pm) {
    p.pm = pm->mode;
    p.tau_pos = pm->tau_pos;
    p.tau_neg = pm->tau_neg;
    if (pm->mode == AA_PM_SAPO) p.rp = AA_F32;  // SAPO's s is fp32 (its temperature tensor is)
  }
  FusedRec *rec = static_cast<FusedRec *>(row_scratch);
  if (entropy) {
    p.entropy = entropy;
    p.ent_coeff = entropy_coeff;
    p.ent_seg = reinterpret_cast<float *>(rec + n_tile_rows);
  }
  if (kl) {
    p.ref = kl->ref;
    p.kl_coeff = kl->coeff;
    p.kl_est = kl->est;
    p.kl_seg = reinterpret_cast<float *>(rec + n_tile_rows) + n_segments;
  }
  return launch_fused(p, logits_dtype, mode, rec, n_tile_rows, static_cast<cudaStream_t>(stream), entropy != nullptr);
}

extern "C" int aa_logprob_actor_fused(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                      const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                      const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                                      const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                                      float *stat_max, float *stat_logsum, const void *old_log_probs, int64_t old_stride,
                                      const void *advantages, int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                                      int64_t mask_stride, int32_t W, float clip_range_ratio, int mode, void *grad_logits,
                                      int64_t grad_row_stride, void *row_scratch, int32_t *status, void *stream) {
  return logprob_actor_fused("aa_logprob_actor_fused", nullptr, 0.f, logits, logits_dtype, row_stride, V, labels, n_segments, seg_logit_off,
                             seg_label_off, seg_out_off, seg_cum, seg_tile_row, n_tile_rows, log_probs, lp_dtype,
                             stat_max, stat_logsum, old_log_probs, old_stride, advantages, adv_stride, adv_dtype, mask,
                             mask_stride, W, clip_range_ratio, clip_range_ratio, 0.f, AA_AGG_SEQ_MEAN_TOKEN_MEAN, mode,
                             grad_logits, grad_row_stride, row_scratch, status, stream);
}

extern "C" int aa_logprob_actor_fused_entropy(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                              const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                              const int64_t *seg_label_off, const int64_t *seg_out_off,
                                              const int64_t *seg_cum, const int64_t *seg_tile_row, int64_t n_tile_rows,
                                              void *log_probs, int lp_dtype, float *stat_max, float *stat_logsum,
                                              const void *old_log_probs, int64_t old_stride, const void *advantages,
                                              int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                                              int64_t mask_stride, int32_t W, float clip_range_ratio, int mode,
                                              void *grad_logits, int64_t grad_row_stride, void *row_scratch,
                                              int32_t *status, float entropy_coeff, float *entropy, void *stream) {
  AA_REQUIRE(entropy, AA_ERR_ARG, "aa_logprob_actor_fused_entropy: null entropy");
  AA_REQUIRE(entropy_coeff == entropy_coeff, AA_ERR_ARG, "aa_logprob_actor_fused_entropy: entropy_coeff is NaN");
  return logprob_actor_fused("aa_logprob_actor_fused_entropy", entropy, entropy_coeff, logits, logits_dtype, row_stride, V, labels, n_segments,
                             seg_logit_off, seg_label_off, seg_out_off, seg_cum, seg_tile_row, n_tile_rows, log_probs,
                             lp_dtype, stat_max, stat_logsum, old_log_probs, old_stride, advantages, adv_stride,
                             adv_dtype, mask, mask_stride, W, clip_range_ratio, clip_range_ratio, 0.f,
                             AA_AGG_SEQ_MEAN_TOKEN_MEAN, mode, grad_logits, grad_row_stride, row_scratch, status, stream);
}

extern "C" int aa_logprob_actor_fused_obj(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                          const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                          const int64_t *seg_label_off, const int64_t *seg_out_off,
                                          const int64_t *seg_cum, const int64_t *seg_tile_row, int64_t n_tile_rows,
                                          void *log_probs, int lp_dtype, float *stat_max, float *stat_logsum,
                                          const void *old_log_probs, int64_t old_stride, const void *advantages,
                                          int64_t adv_stride, int adv_dtype, const uint8_t *mask, int64_t mask_stride,
                                          int32_t W, float clip_low, float clip_high, float dual_clip, int loss_agg,
                                          int mode, void *grad_logits, int64_t grad_row_stride, void *row_scratch,
                                          int32_t *status, float entropy_coeff, float *entropy, void *stream) {
  AA_REQUIRE(actor_objective_ok(clip_low, clip_high, dual_clip, loss_agg), AA_ERR_ARG,
             "aa_logprob_actor_fused_obj: bad objective (need 0 <= clip_low < 1, clip_high >= 0, dual_clip 0 or > 1, a "
             "known loss_agg; got %g %g %g %d)", clip_low, clip_high, dual_clip, loss_agg);
  AA_REQUIRE(entropy_coeff == entropy_coeff, AA_ERR_ARG, "aa_logprob_actor_fused_obj: entropy_coeff is NaN");
  return logprob_actor_fused("aa_logprob_actor_fused_obj", entropy, entropy_coeff, logits, logits_dtype, row_stride, V,
                             labels, n_segments, seg_logit_off, seg_label_off, seg_out_off, seg_cum, seg_tile_row,
                             n_tile_rows, log_probs, lp_dtype, stat_max, stat_logsum, old_log_probs, old_stride,
                             advantages, adv_stride, adv_dtype, mask, mask_stride, W, clip_low, clip_high, dual_clip,
                             loss_agg, mode, grad_logits, grad_row_stride, row_scratch, status, stream);
}

extern "C" int aa_logprob_actor_fused_kl(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                         const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                         const int64_t *seg_label_off, const int64_t *seg_out_off,
                                         const int64_t *seg_cum, const int64_t *seg_tile_row, int64_t n_tile_rows,
                                         void *log_probs, int lp_dtype, float *stat_max, float *stat_logsum,
                                         const void *old_log_probs, int64_t old_stride, const void *advantages,
                                         int64_t adv_stride, int adv_dtype, const uint8_t *mask, int64_t mask_stride,
                                         int32_t W, float clip_low, float clip_high, float dual_clip, int loss_agg,
                                         int mode, void *grad_logits, int64_t grad_row_stride, void *row_scratch,
                                         int32_t *status, float entropy_coeff, float *entropy,
                                         const void *ref_log_probs, float kl_loss_coeff, int kl_estimator,
                                         void *stream) {
  AA_REQUIRE(actor_objective_ok(clip_low, clip_high, dual_clip, loss_agg), AA_ERR_ARG,
             "aa_logprob_actor_fused_kl: bad objective (need 0 <= clip_low < 1, clip_high >= 0, dual_clip 0 or > 1, a "
             "known loss_agg; got %g %g %g %d)", clip_low, clip_high, dual_clip, loss_agg);
  AA_REQUIRE(entropy_coeff == entropy_coeff, AA_ERR_ARG, "aa_logprob_actor_fused_kl: entropy_coeff is NaN");
  AA_REQUIRE(kl_estimator_ok(kl_estimator), AA_ERR_ARG, "aa_logprob_actor_fused_kl: unknown kl_estimator code %d",
             kl_estimator);
  AA_REQUIRE(kl_loss_term_ok(kl_loss_coeff), AA_ERR_ARG,
             "aa_logprob_actor_fused_kl: kl_loss_coeff must be finite and > 0 (got %g)", kl_loss_coeff);
  AA_REQUIRE(ref_log_probs, AA_ERR_ARG, "aa_logprob_actor_fused_kl: null ref_log_probs");
  const ActorKlTerm kl{ref_log_probs, kl_loss_coeff, kl_estimator};
  return logprob_actor_fused("aa_logprob_actor_fused_kl", entropy, entropy_coeff, logits, logits_dtype, row_stride, V,
                             labels, n_segments, seg_logit_off, seg_label_off, seg_out_off, seg_cum, seg_tile_row,
                             n_tile_rows, log_probs, lp_dtype, stat_max, stat_logsum, old_log_probs, old_stride,
                             advantages, adv_stride, adv_dtype, mask, mask_stride, W, clip_low, clip_high, dual_clip,
                             loss_agg, mode, grad_logits, grad_row_stride, row_scratch, status, stream, &kl);
}

extern "C" int aa_logprob_ce_fused(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                  const int64_t *labels, int64_t n_labels, int64_t ignore_index, int32_t n_segments,
                                  const int64_t *seg_logit_off, const int64_t *seg_label_off, const int64_t *seg_out_off,
                                  const int64_t *seg_cum, const int64_t *seg_tile_row, int64_t n_tile_rows,
                                  float *log_probs, float loss_scale, void *grad_logits, int64_t grad_row_stride,
                                  void *row_scratch, float *coeff_scratch, int32_t *status, void *stream) {
  AA_REQUIRE(V > 0 && n_segments > 0 && n_labels > 0 && n_tile_rows > 0 && n_tile_rows % n_segments == 0, AA_ERR_ARG,
             "aa_logprob_ce_fused: bad sizes (the gradient tile holds n_tile_rows / n_segments rows per segment)");
  AA_REQUIRE(logits && labels && seg_logit_off && seg_label_off && seg_out_off && seg_cum && seg_tile_row && log_probs &&
                 grad_logits && row_scratch && coeff_scratch,
             AA_ERR_ARG, "aa_logprob_ce_fused: null pointer");
  AA_REQUIRE(fdtype_ok(logits_dtype), AA_ERR_DTYPE, "aa_logprob_ce_fused: bad dtype");
  AA_REQUIRE((reinterpret_cast<uintptr_t>(row_scratch) & 15) == 0, AA_ERR_ALIGN,
             "aa_logprob_ce_fused: row_scratch must be 16-byte aligned");
  AA_REQUIRE(n_tile_rows < (1ll << 31), AA_ERR_ARG, "aa_logprob_ce_fused: tile too large");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ce_coeff_kernel<<<1, 1024, 0, st>>>(labels, n_labels, ignore_index, loss_scale, coeff_scratch);
  int rc = check_launch("aa_logprob_ce_fused(count)");
  if (rc) return rc;
  FusedActorParams p = fused_params(logits, row_stride, V, labels, n_segments, seg_logit_off, seg_label_off, seg_out_off,
                                    seg_cum, seg_tile_row, n_tile_rows, log_probs, AA_F32, grad_logits,
                                    grad_row_stride, status);
  p.kind = 1;
  p.ignore_index = ignore_index;
  p.ce_coeff = coeff_scratch;
  return launch_fused(p, logits_dtype, AA_MODE_F32, static_cast<FusedRec *>(row_scratch), n_tile_rows, st);
}

// the objective of aa_logprob_grpo_fused_obj (kind 3); pm: the policy loss of aa_logprob_grpo_fused_pm (0: clipped)
struct GrpoObjective {
  const void *old_pol;
  float clip_lo, clip_hi, dual;
  int agg, kl_est;
  PolicyLoss pm;
};

// aa_logprob_grpo_fused{,_entropy,_obj}: entropy == nullptr runs the plain kernels; obj == nullptr: kind 2
static int logprob_grpo_fused(float *entropy, float entropy_coeff, bool egrad, const char *who, const void *logits,
                              int logits_dtype, int64_t row_stride, int32_t V,
                                    const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                    const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                                    const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                                    const void *ref_log_probs, int64_t ref_stride, const float *advantages,
                                    const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t K,
                                    float beta, int mode, void *grad_logits, int64_t grad_row_stride, void *row_scratch,
                                    int32_t *row_end, float *total, uint32_t *counter, int32_t *status, void *stream,
                                    const GrpoObjective *obj = nullptr) {
  AA_REQUIRE(V > 0 && n_segments > 0 && K > 0 && n_tile_rows > 0 && n_tile_rows % n_segments == 0, AA_ERR_ARG,
             "%s: bad sizes (the gradient tile holds n_tile_rows / n_segments rows per sample)", who);
  AA_REQUIRE(logits && labels && seg_logit_off && seg_label_off && seg_out_off && seg_cum && seg_tile_row && log_probs &&
                 ref_log_probs && advantages && completion_tokens && grad_logits && row_scratch && row_end && total && counter,
             AA_ERR_ARG, "%s: null pointer", who);
  AA_REQUIRE(fdtype_ok(logits_dtype) && fdtype_ok(lp_dtype), AA_ERR_DTYPE, "%s: bad dtype", who);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "%s: bad mode", who);
  AA_REQUIRE((reinterpret_cast<uintptr_t>(row_scratch) & 15) == 0, AA_ERR_ALIGN,
             "%s: row_scratch must be 16-byte aligned", who);
  AA_REQUIRE(n_tile_rows < (1ll << 31), AA_ERR_ARG, "%s: tile too large", who);
  const bool f = (mode == AA_MODE_FAITHFUL);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  grpo_mask_kernel<128><<<n_segments, 128, 0, st>>>(completion_tokens, tok_stride, n_segments, K, eos_id, row_end, total, counter);
  int rc = check_launch("aa_logprob_grpo_fused(mask)");
  if (rc) return rc;
  FusedActorParams p = fused_params(logits, row_stride, V, labels, n_segments, seg_logit_off, seg_label_off, seg_out_off,
                                    seg_cum, seg_tile_row, n_tile_rows, log_probs, lp_dtype, grad_logits,
                                    grad_row_stride, status);
  p.kind = 2;
  p.old = ref_log_probs;
  p.old_stride = ref_stride;
  p.adv = advantages;
  p.clip = beta;
  p.rx = f ? lp_dtype : AA_F32;
  p.rp = f ? lp_dtype : AA_F32;
  p.row_end = row_end;
  p.total = total;
  p.entropy = entropy;
  p.ent_coeff = entropy_coeff;
  if (obj) {
    p.kind = 3;
    p.W = K;
    p.old_pol = obj->old_pol;
    p.clip_lo = obj->clip_lo;
    p.clip_hi = obj->clip_hi;
    p.dual = obj->dual;
    p.agg = obj->agg;
    p.kl_est = obj->kl_est;
    p.pm = obj->pm.mode;
    p.tau_pos = obj->pm.tau_pos;
    p.tau_neg = obj->pm.tau_neg;
  }
  return launch_fused(p, logits_dtype, mode, static_cast<FusedRec *>(row_scratch), n_tile_rows, st, egrad);
}

extern "C" int aa_logprob_grpo_fused(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                    const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                    const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                                    const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                                    const void *ref_log_probs, int64_t ref_stride, const float *advantages,
                                    const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t K,
                                    float beta, int mode, void *grad_logits, int64_t grad_row_stride, void *row_scratch,
                                    int32_t *row_end, float *total, uint32_t *counter, int32_t *status, void *stream) {
  return logprob_grpo_fused(nullptr, 0.f, false, "aa_logprob_grpo_fused", logits, logits_dtype, row_stride, V, labels, n_segments,
                            seg_logit_off, seg_label_off, seg_out_off, seg_cum, seg_tile_row, n_tile_rows, log_probs,
                            lp_dtype, ref_log_probs, ref_stride, advantages, completion_tokens, tok_stride, eos_id, K, beta,
                            mode, grad_logits, grad_row_stride, row_scratch, row_end, total, counter, status, stream);
}

extern "C" int aa_logprob_grpo_fused_entropy(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                            const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                            const int64_t *seg_label_off, const int64_t *seg_out_off,
                                            const int64_t *seg_cum, const int64_t *seg_tile_row, int64_t n_tile_rows,
                                            void *log_probs, int lp_dtype, const void *ref_log_probs, int64_t ref_stride,
                                            const float *advantages, const int64_t *completion_tokens, int64_t tok_stride,
                                            int64_t eos_id, int32_t K, float beta, int mode, void *grad_logits,
                                            int64_t grad_row_stride, void *row_scratch, int32_t *row_end, float *total,
                                            uint32_t *counter, int32_t *status, float *entropy, void *stream) {
  AA_REQUIRE(entropy, AA_ERR_ARG, "aa_logprob_grpo_fused_entropy: null entropy");
  return logprob_grpo_fused(entropy, 0.f, false, "aa_logprob_grpo_fused_entropy", logits, logits_dtype, row_stride, V,
                            labels, n_segments, seg_logit_off, seg_label_off, seg_out_off, seg_cum, seg_tile_row,
                            n_tile_rows, log_probs, lp_dtype, ref_log_probs, ref_stride, advantages, completion_tokens,
                            tok_stride, eos_id, K, beta, mode, grad_logits, grad_row_stride, row_scratch, row_end, total,
                            counter, status, stream);
}

extern "C" int aa_logprob_grpo_fused_entropy_grad(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                                 const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                                 const int64_t *seg_label_off, const int64_t *seg_out_off,
                                                 const int64_t *seg_cum, const int64_t *seg_tile_row, int64_t n_tile_rows,
                                                 void *log_probs, int lp_dtype, const void *ref_log_probs,
                                                 int64_t ref_stride, const float *advantages,
                                                 const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id,
                                                 int32_t K, float beta, int mode, void *grad_logits,
                                                 int64_t grad_row_stride, void *row_scratch, int32_t *row_end,
                                                 float *total, uint32_t *counter, int32_t *status, float *entropy,
                                                 float entropy_coeff, void *stream) {
  AA_REQUIRE(entropy, AA_ERR_ARG, "aa_logprob_grpo_fused_entropy_grad: null entropy");
  AA_REQUIRE(entropy_coeff == entropy_coeff, AA_ERR_ARG, "aa_logprob_grpo_fused_entropy_grad: entropy_coeff is NaN");
  return logprob_grpo_fused(entropy, entropy_coeff, true, "aa_logprob_grpo_fused_entropy_grad", logits, logits_dtype,
                            row_stride, V, labels, n_segments, seg_logit_off, seg_label_off, seg_out_off, seg_cum,
                            seg_tile_row, n_tile_rows, log_probs, lp_dtype, ref_log_probs, ref_stride, advantages,
                            completion_tokens, tok_stride, eos_id, K, beta, mode, grad_logits, grad_row_stride,
                            row_scratch, row_end, total, counter, status, stream);
}

// aa_logprob_grpo_fused_obj / _kl: the objective's checks, then kind 3
static int logprob_grpo_fused_objective(const char *who, const void *logits, int logits_dtype, int64_t row_stride,
                                        int32_t V, const int64_t *labels, int32_t n_segments,
                                        const int64_t *seg_logit_off, const int64_t *seg_label_off,
                                        const int64_t *seg_out_off, const int64_t *seg_cum, const int64_t *seg_tile_row,
                                        int64_t n_tile_rows, void *log_probs, int lp_dtype, const void *ref_log_probs,
                                        int64_t ref_stride, const void *old_log_probs, const float *advantages,
                                        const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t K,
                                        float beta, float clip_low, float clip_high, float dual_clip, int loss_agg,
                                        int kl_estimator, int mode, void *grad_logits, int64_t grad_row_stride,
                                        void *row_scratch, int32_t *row_end, float *total, uint32_t *counter,
                                        int32_t *status, float *entropy, float entropy_coeff, void *stream,
                                        PolicyLoss pm = PolicyLoss{0, 1.f, 1.f}) {
  AA_REQUIRE(grpo_objective_ok(clip_low, clip_high, dual_clip, loss_agg), AA_ERR_ARG,
             "%s: bad objective (need 0 <= clip_low < 1, clip_high >= 0, dual_clip 0 or > 1, a known loss_agg; got %g "
             "%g %g %d)", who, clip_low, clip_high, dual_clip, loss_agg);
  AA_REQUIRE(kl_estimator_ok(kl_estimator), AA_ERR_ARG, "%s: unknown kl_estimator code %d", who, kl_estimator);
  AA_REQUIRE(entropy_coeff == entropy_coeff, AA_ERR_ARG, "%s: entropy_coeff is NaN", who);
  AA_REQUIRE(entropy || entropy_coeff == 0.f, AA_ERR_ARG, "%s: entropy_coeff needs entropy", who);
  GrpoObjective obj{old_log_probs, clip_low, clip_high, dual_clip, loss_agg, kl_estimator, pm};
  return logprob_grpo_fused(entropy, entropy_coeff, entropy && entropy_coeff != 0.f, who, logits, logits_dtype,
                            row_stride, V, labels, n_segments, seg_logit_off, seg_label_off, seg_out_off, seg_cum,
                            seg_tile_row, n_tile_rows, log_probs, lp_dtype, ref_log_probs, ref_stride, advantages,
                            completion_tokens, tok_stride, eos_id, K, beta, mode, grad_logits, grad_row_stride,
                            row_scratch, row_end, total, counter, status, stream, &obj);
}

extern "C" int aa_logprob_grpo_fused_obj(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                         const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                         const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                                         const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                                         const void *ref_log_probs, int64_t ref_stride, const void *old_log_probs,
                                         const float *advantages, const int64_t *completion_tokens, int64_t tok_stride,
                                         int64_t eos_id, int32_t K, float beta, float clip_low, float clip_high,
                                         float dual_clip, int loss_agg, int mode, void *grad_logits,
                                         int64_t grad_row_stride, void *row_scratch, int32_t *row_end, float *total,
                                         uint32_t *counter, int32_t *status, float *entropy, float entropy_coeff,
                                         void *stream) {
  return logprob_grpo_fused_objective("aa_logprob_grpo_fused_obj", logits, logits_dtype, row_stride, V, labels,
                                      n_segments, seg_logit_off, seg_label_off, seg_out_off, seg_cum, seg_tile_row,
                                      n_tile_rows, log_probs, lp_dtype, ref_log_probs, ref_stride, old_log_probs,
                                      advantages, completion_tokens, tok_stride, eos_id, K, beta, clip_low, clip_high,
                                      dual_clip, loss_agg, AA_KL_K3, mode, grad_logits, grad_row_stride, row_scratch,
                                      row_end, total, counter, status, entropy, entropy_coeff, stream);
}

extern "C" int aa_logprob_grpo_fused_kl(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                        const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                        const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                                        const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                                        const void *ref_log_probs, int64_t ref_stride, const void *old_log_probs,
                                        const float *advantages, const int64_t *completion_tokens, int64_t tok_stride,
                                        int64_t eos_id, int32_t K, float beta, float clip_low, float clip_high,
                                        float dual_clip, int loss_agg, int kl_estimator, int mode, void *grad_logits,
                                        int64_t grad_row_stride, void *row_scratch, int32_t *row_end, float *total,
                                        uint32_t *counter, int32_t *status, float *entropy, float entropy_coeff,
                                        void *stream) {
  return logprob_grpo_fused_objective("aa_logprob_grpo_fused_kl", logits, logits_dtype, row_stride, V, labels,
                                      n_segments, seg_logit_off, seg_label_off, seg_out_off, seg_cum, seg_tile_row,
                                      n_tile_rows, log_probs, lp_dtype, ref_log_probs, ref_stride, old_log_probs,
                                      advantages, completion_tokens, tok_stride, eos_id, K, beta, clip_low, clip_high,
                                      dual_clip, loss_agg, kl_estimator, mode, grad_logits, grad_row_stride,
                                      row_scratch, row_end, total, counter, status, entropy, entropy_coeff, stream);
}

extern "C" int aa_logprob_actor_fused_pm(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                         const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                         const int64_t *seg_label_off, const int64_t *seg_out_off,
                                         const int64_t *seg_cum, const int64_t *seg_tile_row, int64_t n_tile_rows,
                                         void *log_probs, int lp_dtype, float *stat_max, float *stat_logsum,
                                         const void *old_log_probs, int64_t old_stride, const void *advantages,
                                         int64_t adv_stride, int adv_dtype, const uint8_t *mask, int64_t mask_stride,
                                         int32_t W, float clip_high, int loss_agg, int pm_mode, float tau_pos,
                                         float tau_neg, int mode, void *grad_logits, int64_t grad_row_stride,
                                         void *row_scratch, int32_t *status, float entropy_coeff, float *entropy,
                                         const void *ref_log_probs, float kl_loss_coeff, int kl_estimator,
                                         void *stream) {
  const char *who = "aa_logprob_actor_fused_pm";
  AA_REQUIRE(pm_mode_ok(pm_mode), AA_ERR_ARG, "%s: unknown pm_mode %d", who, pm_mode);
  AA_REQUIRE(actor_objective_ok(0.f, clip_high, 0.f, loss_agg), AA_ERR_ARG,
             "%s: bad objective (need clip_high >= 0 and a known loss_agg; got %g %d)", who, clip_high, loss_agg);
  AA_REQUIRE(sapo_temperature_ok(tau_pos) && sapo_temperature_ok(tau_neg), AA_ERR_ARG,
             "%s: tau_pos and tau_neg must be finite and > 0 (got %g %g)", who, tau_pos, tau_neg);
  AA_REQUIRE(entropy_coeff == entropy_coeff, AA_ERR_ARG, "%s: entropy_coeff is NaN", who);
  AA_REQUIRE(entropy || entropy_coeff == 0.f, AA_ERR_ARG, "%s: entropy_coeff needs entropy", who);
  if (ref_log_probs) {
    AA_REQUIRE(kl_estimator_ok(kl_estimator), AA_ERR_ARG, "%s: unknown kl_estimator code %d", who, kl_estimator);
    AA_REQUIRE(kl_loss_term_ok(kl_loss_coeff), AA_ERR_ARG, "%s: kl_loss_coeff must be finite and > 0 (got %g)", who,
               kl_loss_coeff);
  }
  const ActorKlTerm kl{ref_log_probs, kl_loss_coeff, kl_estimator};
  const PolicyLoss pm{pm_mode, tau_pos, tau_neg};
  return logprob_actor_fused(who, entropy, entropy_coeff, logits, logits_dtype, row_stride, V, labels, n_segments,
                             seg_logit_off, seg_label_off, seg_out_off, seg_cum, seg_tile_row, n_tile_rows, log_probs,
                             lp_dtype, stat_max, stat_logsum, old_log_probs, old_stride, advantages, adv_stride,
                             adv_dtype, mask, mask_stride, W, 0.f, clip_high, 0.f, loss_agg, mode, grad_logits,
                             grad_row_stride, row_scratch, status, stream, ref_log_probs ? &kl : nullptr, &pm);
}

extern "C" int aa_logprob_grpo_fused_pm(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                        const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                        const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                                        const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                                        const void *ref_log_probs, int64_t ref_stride, const void *old_log_probs,
                                        const float *advantages, const int64_t *completion_tokens, int64_t tok_stride,
                                        int64_t eos_id, int32_t K, float beta, float clip_high, int loss_agg,
                                        int kl_estimator, int pm_mode, float tau_pos, float tau_neg, int mode,
                                        void *grad_logits, int64_t grad_row_stride, void *row_scratch,
                                        int32_t *row_end, float *total, uint32_t *counter, int32_t *status,
                                        float *entropy, float entropy_coeff, void *stream) {
  AA_REQUIRE(pm_mode_ok(pm_mode), AA_ERR_ARG, "aa_logprob_grpo_fused_pm: unknown pm_mode %d", pm_mode);
  AA_REQUIRE(sapo_temperature_ok(tau_pos) && sapo_temperature_ok(tau_neg), AA_ERR_ARG,
             "aa_logprob_grpo_fused_pm: tau_pos and tau_neg must be finite and > 0 (got %g %g)", tau_pos, tau_neg);
  return logprob_grpo_fused_objective("aa_logprob_grpo_fused_pm", logits, logits_dtype, row_stride, V, labels,
                                      n_segments, seg_logit_off, seg_label_off, seg_out_off, seg_cum, seg_tile_row,
                                      n_tile_rows, log_probs, lp_dtype, ref_log_probs, ref_stride, old_log_probs,
                                      advantages, completion_tokens, tok_stride, eos_id, K, beta, 0.f, clip_high, 0.f,
                                      loss_agg, kl_estimator, mode, grad_logits, grad_row_stride, row_scratch,
                                      row_end, total, counter, status, entropy, entropy_coeff, stream,
                                      PolicyLoss{pm_mode, tau_pos, tau_neg});
}

extern "C" int aa_scale_tile(void *tile, int dtype, int64_t n, const void *scale, int scale_dtype, void *stream) {
  AA_REQUIRE(n >= 0 && fdtype_ok(dtype) && fdtype_ok(scale_dtype), AA_ERR_ARG, "aa_scale_tile: bad arguments");
  if (n == 0) return AA_OK;
  AA_REQUIRE(tile && scale, AA_ERR_ARG, "aa_scale_tile: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned grid = static_cast<unsigned>(sm_count()) * 8u;
  switch (dtype) {
    case AA_BF16: scale_tile_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(static_cast<__nv_bfloat16 *>(tile), n, scale, scale_dtype); break;
    case AA_F16: scale_tile_kernel<__half><<<grid, 256, 0, st>>>(static_cast<__half *>(tile), n, scale, scale_dtype); break;
    default: scale_tile_kernel<float><<<grid, 256, 0, st>>>(static_cast<float *>(tile), n, scale, scale_dtype);
  }
  return check_launch("aa_scale_tile");
}
