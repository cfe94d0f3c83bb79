// linear_logprob.cu -- K6 (SURVEY.md 8f rank 1): lm_head x log-prob in ONE kernel, no (rows, V) logits tile.
//
//   logp[r] = log_softmax(hidden[r, :] @ weight^T)[label[r]]          hidden (N, H) bf16, weight (V, H) bf16
//
// i.e. `gather_log_probabilities(lm_head(hidden), labels)` (utils/tools.py:402-413 on the output of the
// model's nn.Linear lm_head, callers trainers/text_to_text/dpo.py:128, ppo.py:266-267) for rows that carry no
// gradient (reference model, rollout scoring).  The GEMM runs on the Hopper tensor cores (wgmma.cuh):
//
//   warpgroup 2  : TMA producer -- cp.async.bulk.tensor 2-D boxes (64 x 128 of hidden, 64 x 256 of weight, 128-byte
//                  swizzle) into a 4-stage shared-memory ring, mbarrier expect_tx / complete_tx
//   warpgroups 0-1: wgmma m64n256k16 (bf16 x bf16 -> fp32 registers), 64 rows each, then the epilogue on the
//                  registers: round to bf16 (the rounding point of the reference's nn.Linear), online (max, sum-exp)
//                  update, label-column pick.  The producer keeps filling the ring while the epilogue runs.
//
// One CTA owns 128 rows and sweeps the whole vocabulary (or a split of it), so (max, sum) never leave registers;
// concurrently running CTAs sweep the weight in step, which keeps it L2-resident.
// Both operands are K-major with 16-byte aligned rows (H * 2 bytes), so TMA applies although V = 128257 is odd:
// the odd leading dimension only ever existed in the logits tile, which is never written here.
#include <atomic>

#include "wgmma.cuh"

namespace aa {
namespace k6 {

using namespace wg;  // BM / BN / BK, mbarrier + TMA + wgmma wrappers, descriptors (shared with linear_backward.cu)

struct Params {
  const int64_t *labels;
  int64_t n_rows;
  int V, H;
  void *out;
  int out_dtype;
  float *stat_max, *stat_logsum;
  int faithful;
  int32_t *status;
  int v_splits, tiles_per_split;  // blockIdx.y sweeps vocabulary tiles [y * tiles_per_split, ...)
  int rot_groups;                 // CTAs start their sweep (m_tile % rot_groups) * rot_step tiles into the range
  int rot_step;
  int group_tiles, m_tiles;       // linear block id -> (row-tile group, split, row tile in group); see the host code
  float *partial;                 // v_splits > 1: (row, split) -> {max, sum, label logit[, entropy sum t]}
  float *entropy;                 // ENT kernels: fp32 entropy per row
};

// the tile store of K6b (d(logits)) and K6s (the logits): the upstream gradient per row (K6b) and the padded bf16 buffer
struct GradParams {
  const void *grad_rows;  // upstream d loss / d logp per row
  int grad_rows_dtype;
  __nv_bfloat16 *dlogits; // (n_rows, ld) bf16, ld >= ceil(V / 256) * 256, multiple of 8
  int64_t ld;
  // K6b's entropy-gradient kernel (ENT): the upstream gradient of each row's entropy (dtype grad_entropy_dtype); the
  // entropy itself is read from Params::entropy (K6's entropy variant wrote it)
  const void *grad_entropy;
  int grad_entropy_dtype;
};

// what the consumer warpgroups do with a finished 128 x 256 logits tile
enum class Epi : int {
  Lse,      // K6: fold it into the row's running (max, sum-exp, label logit)
  DLogits,  // K6b: turn it into d(logits) with the statistics K6 saved and store it
  Logits,   // K6s: both K6's fold and a store of the bf16-rounded logits
};

__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// merge two partial (max, sum-exp) of one row
__device__ __forceinline__ void lse_merge(float &m, float &s, float m_o, float s_o) {
  const float mn = fmaxf(m, m_o);
  if (mn == -INFINITY) return;  // both empty: s == s_o == 0
  s = (m == -INFINITY ? 0.f : s * ex2_approx((m - mn) * kLog2e)) + (m_o == -INFINITY ? 0.f : s_o * ex2_approx((m_o - mn) * kLog2e));
  m = mn;
}

// the same with the entropy sum t = sum e^{x - m} (x - m) (logprob_math.cuh: t' = alpha (t + (m - m') s)); the (m, s)
// arithmetic is lse_merge's, so the statistics do not depend on whether the entropy is on
__device__ __forceinline__ float ent_part(float t, float s, float m, float mn) {
  return m == -INFINITY ? 0.f : (m == mn ? t : ex2_approx((m - mn) * kLog2e) * fmaf(m - mn, s, t));
}
__device__ __forceinline__ void lse_merge_ent(float &m, float &s, float &t, float m_o, float s_o, float t_o) {
  const float mn = fmaxf(m, m_o);
  if (mn == -INFINITY) return;
  t = ent_part(t, s, m, mn) + ent_part(t_o, s_o, m_o, mn);
  lse_merge(m, s, m_o, s_o);
}

// K6, K6b and K6s are ONE kernel: same TMA producer, same wgmma main loop; they differ in what the consumer
// warpgroups do with a finished 128 x 256 logits tile (Epi) -- fold it into the running (max, sum-exp, label logit) of
// the row, turn it into d(logits) with the statistics K6 saved and store it as bf16, or (K6s) fold it AND store the
// bf16-rounded logits, so that the logits of a loss whose gradient seed is known in the forward cost one GEMM pass.
// Each consumer thread holds 2 rows x 64 columns of the tile (wgmma.cuh, frag_row / frag_col); the 4 threads of a quad
// share a row, so the per-row statistics are per-thread partials merged across the quad once, at the end.
template <Epi EPI, bool ENT = false>
__global__ void __launch_bounds__(THREADS, 1)
    linear_logprob_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                          const Params p, const GradParams gp) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t *full = reinterpret_cast<uint64_t *>(tiles + STAGES * STAGE_BYTES);
  uint64_t *empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // block id -> (group of `group_tiles` row tiles) x (vocabulary split) x (row tile in the group): the CTAs that are
  // resident together work on few row tiles (their hidden-state tiles, 1 MB each and re-read for every vocabulary
  // tile, must stay in L2 next to the weight tiles of the moment) and on all splits of those rows
  const int unit = static_cast<int>(blockIdx.x);
  const int per_group = p.group_tiles * p.v_splits;
  const int grp = unit / per_group, rem = unit % per_group;
  const int m_unit = grp * p.group_tiles + rem % p.group_tiles;
  const int split = rem / p.group_tiles;
  if (m_unit >= p.m_tiles) return;  // tail of the last group (uniform per CTA, before any barrier use)
  const int m0 = m_unit * BM;
  const int all_tiles = (p.V + BN - 1) / BN;
  const int t0 = split * p.tiles_per_split;
  const int n_tiles = min(all_tiles - t0, p.tiles_per_split);  // >= 1 by construction of the grid
  const int k_blocks = p.H / BK;
  // The online softmax is order independent, so every CTA may sweep its vocabulary range from a different start:
  // at any moment `rot_groups` different weight tiles are hot in L2 instead of one that all SMs hammer.  Every launch
  // passes rot_groups = 1 (no rotation).  The term stays because ptxas schedules the kernel differently without it:
  // K6 ran 7 % slower on an H100 80GB HBM3 at 400 W (C2 shapes, 34.6 ms against 32.3 ms).
  const int rot = (p.rot_groups > 1) ? static_cast<int>((m_unit % p.rot_groups) * p.rot_step) % n_tiles : 0;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(full + i, 1);
      mbar_init(empty + i, CONSUMER_THREADS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (threadIdx.x >= CONSUMER_THREADS) {
    // ------------------------------- TMA producer -------------------------------
    producer_regs();
    if (warp == CONSUMER_THREADS / 32 && lane == 0) {
      int64_t it = 0;
      for (int nt = 0; nt < n_tiles; ++nt) {
        const int v_row0 = (t0 + (nt + rot) % n_tiles) * BN;
        for (int kb = 0; kb < k_blocks; ++kb, ++it) {
          const int s = static_cast<int>(it % STAGES);
          mbar_wait(empty + s, static_cast<uint32_t>((it / STAGES) & 1) ^ 1u);
          uint8_t *a = tiles + s * STAGE_BYTES, *b = a + A_BYTES;
          mbar_expect_tx(full + s, STAGE_BYTES);
          tma_load_2d(a, &map_a, kb * BK, m0, full + s);
          tma_load_2d(b, &map_b, kb * BK, v_row0, full + s);
        }
      }
    }
    return;
  }

  // ------------------------------- consumers: wgmma + epilogue ----------------------------
  consumer_regs();
  const int w = threadIdx.x >> 7, t = threadIdx.x & 127;
  int64_t row[2], label[2];
  bool live[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    row[r] = static_cast<int64_t>(m0) + 64 * w + frag_row(t, 2 * r);
    live[r] = row[r] < p.n_rows;
    label[r] = live[r] ? __ldg(p.labels + row[r]) : -1;
  }
  float acc[ACC];
  int64_t it = 0;
  if constexpr (EPI != Epi::DLogits) {
    // ------------------------------- K6 / K6s epilogue: online log-sum-exp ----------------
    // K6s rounds every logit to bf16 whatever the mode (the stored tile is bf16, and the statistics must describe it);
    // the mode then only decides whether the log-prob is rounded.  K6s's pad columns of the last tile are stored as +0.
    __nv_bfloat16 *lrow[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) lrow[r] = gp.dlogits + (live[r] ? row[r] : 0) * gp.ld;
    if ((t & 3) == 0 && p.status) {
#pragma unroll
      for (int r = 0; r < 2; ++r)
        if (live[r] && (label[r] < 0 || label[r] >= p.V)) atomicOr(p.status, AA_STATUS_LABEL_OOB);
    }
    // label column as an index into the tile's columns held by this thread (out of range: never matches)
    int lab[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) lab[r] = (label[r] >= 0 && label[r] < p.V) ? static_cast<int>(label[r]) : -BN;
    float m[2] = {-INFINITY, -INFINITY}, s[2] = {0.f, 0.f}, x_label[2] = {-INFINITY, -INFINITY};
    float ent_t[2] = {0.f, 0.f};  // ENT: running sum e^{x - m} (x - m) of the values the statistics fold
    for (int nt = 0; nt < n_tiles; ++nt) {
      consume_tile<0, 0>(acc, tiles, full, empty, k_blocks, it, w);
      const int col_base = (t0 + (nt + rot) % n_tiles) * BN;
      if (col_base + BN > p.V) {  // vocabulary tail (TMA zero-filled the rows)
#pragma unroll
        for (int i = 0; i < ACC; ++i)
          if (col_base + frag_col(t, i) >= p.V) acc[i] = -INFINITY;
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        // label column: a select over the thread's columns rather than a branch (the accumulators must not be read
        // in divergent code, or ptxas serialises the wgmmas)
        const int rel = lab[r] - col_base - 2 * (t & 3);  // = 8 * (i / 4) + i % 2 for the matching i
#pragma unroll
        for (int i = 2 * r; i < ACC; i += 4) {
          x_label[r] = (rel == frag_col(0, i)) ? acc[i] : x_label[r];
          x_label[r] = (rel == frag_col(0, i + 1)) ? acc[i + 1] : x_label[r];
        }
        // FAITHFUL: every logit is rounded to bf16 (nn.Linear returns bf16) where it is used, not in place (writing
        // the accumulators here costs the wgmma pipeline its registers); rounding is monotonic, so the maximum of
        // the rounded logits is the rounded maximum
        float cmax = -INFINITY;
#pragma unroll
        for (int i = 2 * r; i < ACC; i += 4) cmax = fmaxf(cmax, fmaxf(acc[i], acc[i + 1]));
        if (EPI == Epi::Logits || p.faithful) cmax = bf16_round(cmax);
        if (cmax > m[r]) {  // m == -inf implies s == 0
          if constexpr (ENT) {
            if (m[r] != -INFINITY) ent_t[r] = ex2_approx((m[r] - cmax) * kLog2e) * fmaf(m[r] - cmax, s[r], ent_t[r]);
          }
          s[r] *= ex2_approx((m[r] - cmax) * kLog2e);
          m[r] = cmax;
        }
        float add = 0.f, tadd = 0.f;
#pragma unroll
        for (int i = 2 * r; i < ACC; i += 4) {
          float x0 = acc[i], x1 = acc[i + 1];
          if constexpr (EPI == Epi::Logits) {  // ONE rounding serves the store and the fold
            const uint32_t w = pack2<__nv_bfloat16>(x0, x1);
            unpack2<__nv_bfloat16>(w, x0, x1);
            const int col = col_base + frag_col(t, i);
            if (live[r])
              *reinterpret_cast<uint32_t *>(lrow[r] + col) = col + 1 < p.V ? w : (col < p.V ? (w & 0xffffu) : 0u);
          } else {
            if (p.faithful) round_bf16_pair(x0, x1);
          }
          if constexpr (ENT) {
            // pad columns of the last tile are -inf: their (x - m) is clamped so that the term is 0 * finite
            const float d0 = x0 - m[r], d1 = x1 - m[r];
            const float e0 = ex2_approx(d0 * kLog2e), e1 = ex2_approx(d1 * kLog2e);
            add += e0 + e1;
            tadd = fmaf(e0, fmaxf(d0, -3.0e38f), fmaf(e1, fmaxf(d1, -3.0e38f), tadd));
          } else {
            add += ex2_approx((x0 - m[r]) * kLog2e) + ex2_approx((x1 - m[r]) * kLog2e);
          }
        }
        s[r] += add;
        if constexpr (ENT) ent_t[r] += tadd;
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if (EPI == Epi::Logits || p.faithful) x_label[r] = bf16_round(x_label[r]);
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        const float m_o = __shfl_xor_sync(0xffffffffu, m[r], o), s_o = __shfl_xor_sync(0xffffffffu, s[r], o);
        x_label[r] = fmaxf(x_label[r], __shfl_xor_sync(0xffffffffu, x_label[r], o));
        if constexpr (ENT) {
          lse_merge_ent(m[r], s[r], ent_t[r], m_o, s_o, __shfl_xor_sync(0xffffffffu, ent_t[r], o));
        } else {
          lse_merge(m[r], s[r], m_o, s_o);
        }
      }
      if ((t & 3) != 0 || !live[r]) continue;
      if (p.v_splits > 1) {
        float *dst = p.partial + (row[r] * p.v_splits + split) * (ENT ? 4 : 3);
        dst[0] = m[r];
        dst[1] = s[r];
        dst[2] = x_label[r];
        if constexpr (ENT) dst[3] = ent_t[r];
      } else {
        const float logsum = logf(s[r]);
        float lp = (x_label[r] - m[r]) - logsum;
        if (label[r] < 0 || label[r] >= p.V) lp = __int_as_float(0x7fc00000);
        if (p.faithful) lp = __bfloat162float(__float2bfloat16_rn(lp));
        store_from_float(p.out, row[r], p.out_dtype, lp);
        if (p.stat_max) p.stat_max[row[r]] = m[r];
        if (p.stat_logsum) p.stat_logsum[row[r]] = logsum;
        if constexpr (ENT) p.entropy[row[r]] = logsum - ent_t[r] / s[r];
      }
    }
  } else {
    // ------------------------------- K6b epilogue: d(logits) tile store ----------------
    // d(logits)[row, col] = g * ([col == label] - p),  p = exp(round_bf16((x - max) - logsum)) in FAITHFUL mode
    // (what ATen's backward sees: it re-reads the rounded log-softmax), written as bf16 into the padded buffer
    // ENT: a row whose entropy has the upstream gradient g_H gets - g_H p (l + H) added in fp32 before the bf16 store,
    // with the p and l of the line above (logprob_math.cuh, vec_grad_ent); rows with g_H == 0 keep the plain bits
    // (a select, not a branch: the accumulators must not be read in divergent code)
    float m[2], logsum[2], g[2], h[2] = {0.f, 0.f}, ngh[2] = {0.f, 0.f};
    __nv_bfloat16 *drow[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      m[r] = live[r] ? __ldg(p.stat_max + row[r]) : 0.f;
      logsum[r] = live[r] ? __ldg(p.stat_logsum + row[r]) : 0.f;
      g[r] = live[r] ? load_as_float(gp.grad_rows, row[r], gp.grad_rows_dtype) : 0.f;
      drow[r] = gp.dlogits + (live[r] ? row[r] : 0) * gp.ld;
      if constexpr (ENT) {
        h[r] = live[r] ? __ldg(p.entropy + row[r]) : 0.f;
        ngh[r] = live[r] ? -load_as_float(gp.grad_entropy, row[r], gp.grad_entropy_dtype) : 0.f;
      }
    }
    for (int nt = 0; nt < n_tiles; ++nt) {
      consume_tile<0, 0>(acc, tiles, full, empty, k_blocks, it, w);
      const int col_base = (t0 + (nt + rot) % n_tiles) * BN;
#pragma unroll
      for (int i = 0; i < ACC; i += 2) {
        const int r = (i >> 1) & 1;
        const int col = col_base + frag_col(t, i);
        float xs[2] = {acc[i], acc[i + 1]};
        if (p.faithful) round_bf16_pair(xs[0], xs[1]);
        float ls[2] = {(xs[0] - m[r]) - logsum[r], (xs[1] - m[r]) - logsum[r]};
        if (p.faithful) round_bf16_pair(ls[0], ls[1]);
        const float e0 = ex2_approx(ls[0] * kLog2e), e1 = ex2_approx(ls[1] * kLog2e);
        float d0 = e0 * -g[r];  // -(p * g), every column but the label's
        float d1 = e1 * -g[r];
        if (label[r] == col) d0 = __fadd_rn(d0, g[r]);  // g - p * g, the same two roundings
        if (label[r] == col + 1) d1 = __fadd_rn(d1, g[r]);
        if constexpr (ENT) {
          const float c0 = fmaf(e0 * (fmaxf(ls[0], -3.0e38f) + h[r]), ngh[r], d0);
          const float c1 = fmaf(e1 * (fmaxf(ls[1], -3.0e38f) + h[r]), ngh[r], d1);
          d0 = ngh[r] != 0.f ? c0 : d0;
          d1 = ngh[r] != 0.f ? c1 : d1;
        }
        if (col >= p.V) d0 = 0.f;  // last vocabulary tile: pad columns of the buffer stay zero
        if (col + 1 >= p.V) d1 = 0.f;
        if (live[r]) *reinterpret_cast<uint32_t *>(drow[r] + col) = pack2<__nv_bfloat16>(d0, d1);
      }
    }
  }
}

// v_splits > 1: merge the per-split (max, sum, label logit[, entropy sum]) of each row
template <bool ENT = false>
__global__ void linear_logprob_merge_kernel(const Params p) {
  constexpr int F = ENT ? 4 : 3;  // floats per (row, split)
  const int64_t row = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (row >= p.n_rows) return;
  const float *src = p.partial + row * p.v_splits * F;
  float m = -INFINITY, x_label = -INFINITY;
  for (int i = 0; i < p.v_splits; ++i) {
    m = fmaxf(m, src[F * i]);
    x_label = fmaxf(x_label, src[F * i + 2]);  // exactly one split holds the label column
  }
  float s = 0.f;
  for (int i = 0; i < p.v_splits; ++i) s += src[F * i + 1] * ex2_approx((src[F * i] - m) * kLog2e);
  if constexpr (ENT) {  // t = sum_i alpha_i (t_i + (m_i - m) s_i), alpha_i = e^{m_i - m}
    float t = 0.f;
    for (int i = 0; i < p.v_splits; ++i) t += ent_part(src[F * i + 3], src[F * i + 1], src[F * i], m);
    p.entropy[row] = logf(s) - t / s;
  }
  const int64_t label = __ldg(p.labels + row);
  const float logsum = logf(s);
  float lp = (x_label - m) - logsum;
  if (label < 0 || label >= p.V) lp = __int_as_float(0x7fc00000);
  if (p.faithful) lp = __bfloat162float(__float2bfloat16_rn(lp));
  store_from_float(p.out, row, p.out_dtype, lp);
  if (p.stat_max) p.stat_max[row] = m;
  if (p.stat_logsum) p.stat_logsum[row] = logsum;
}

// (rows, H) bf16 row-major -> boxes of 64 (K) x box_rows, 128-byte swizzle, out-of-range rows read as zero
static int make_map(CUtensorMap *map, const void *base, int64_t rows, int H, int64_t row_stride, int box_rows) {
  return make_map_2d(map, base, H, rows, row_stride, box_rows, "aa_linear_logprob_fwd");
}

// ---- host: scheduling and launch shared by K6 / K6b / K6s -----------------------------------------------------------
// One CTA owns 128 rows x a range of vocabulary tiles and keeps (max, sum) in registers.  The L2 working set decides
// the speed: the 1 MB hidden-state tile of every resident CTA is re-read for each vocabulary tile, and all of them plus
// the weight tiles do not fit the 50 MB L2.  So the resident wave is shaped as `group` row units x `splits` vocabulary
// ranges: with S resident CTAs, about S/12 row units keep ~11 MB of hidden tiles hot and each weight tile is shared by
// as many units; with fewer row units than S/8 the vocabulary is spread over the idle SMs.
struct Schedule {
  int64_t splits, group, n_groups, units;
  int tps;
};
static Schedule make_schedule(int64_t n_rows, int V, bool may_split, int64_t partial_floats, int per_split = 3) {
  const int rows_per_unit = BM;
  const int S = sm_count();
  Schedule sc;
  sc.units = (n_rows + rows_per_unit - 1) / rows_per_unit;
  const int all_tiles = (V + BN - 1) / BN;
  sc.splits = 1;
  sc.group = sc.units;
  if (may_split) {
    if (sc.units < S / 8) {
      sc.splits = S / sc.units;
    } else {
      // Every live unit does the same work (tiles-per-split vocabulary tiles), so the kernel takes
      // ceil(units * splits / S) rounds of `tps` tiles: pick the split count around 12 that wastes the least of the
      // last round.  The resident wave holds all splits of S / splits row tiles: ~11 hidden-state tiles and ~12 weight
      // tiles share the 50 MB L2.  (H100, 16 376 rows, H = 4096, V = 128257: 12 x 11 and 16 x 8 both ran 32.9 ms,
      // 8 x 16 35.4 ms, 4 x 33 41.4 ms, 1 x 132 45.0 ms.)
      int64_t best = 12, best_cost = INT64_MAX;
      for (int64_t s = 6; s <= 16; ++s) {
        const int64_t tps = (all_tiles + s - 1) / s;
        const int64_t live = sc.units * ((all_tiles + tps - 1) / tps);
        const int64_t cost = ((live + S - 1) / S) * tps * 64 + (s > 12 ? s - 12 : 12 - s);  // rounds x tiles, ties -> 12
        if (cost < best_cost) best_cost = cost, best = s;
      }
      sc.splits = best;
      sc.group = S / sc.splits;
    }
    if (sc.splits > all_tiles) sc.splits = all_tiles;
    if (sc.splits < 1) sc.splits = 1;
    while (partial_floats >= 0 && sc.splits > 1 && n_rows * sc.splits * per_split > partial_floats) --sc.splits;
    if (sc.group > sc.units) sc.group = sc.units;
    if (sc.group < 1) sc.group = 1;
  }
  sc.tps = static_cast<int>((all_tiles + sc.splits - 1) / sc.splits);
  sc.splits = (all_tiles + sc.tps - 1) / sc.tps;  // no empty split
  sc.n_groups = (sc.units + sc.group - 1) / sc.group;
  return sc;
}

template <Epi EPI, bool ENT = false>
static int launch(const void *hidden, int64_t n_rows, int H, int64_t hidden_row_stride, const void *weight, int V,
                  int64_t weight_row_stride, Params p, const GradParams &gp, const Schedule &sc, cudaStream_t st,
                  const char *who) {
  CUtensorMap map_a, map_b;
  int rc = make_map(&map_a, hidden, n_rows, H, hidden_row_stride, BM);
  if (rc) return rc;
  rc = make_map(&map_b, weight, V, H, weight_row_stride, BN);
  if (rc) return rc;
  p.v_splits = static_cast<int>(sc.splits);
  p.tiles_per_split = sc.tps;
  p.group_tiles = static_cast<int>(sc.group);
  p.m_tiles = static_cast<int>(sc.units);
  const unsigned units = static_cast<unsigned>(sc.n_groups * sc.group * sc.splits);
  auto kern = linear_logprob_kernel<EPI, ENT>;
  static std::atomic<bool> configured{false};  // once per process (idempotent; a race sets it twice, harmlessly)
  if (!configured.load(std::memory_order_relaxed)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) {
      set_error("%s: %s", who, cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    configured.store(true, std::memory_order_relaxed);
  }
  kern<<<units, THREADS, SMEM_BYTES, st>>>(map_a, map_b, p, gp);
  return check_launch(who);
}

// K6 / K6s: argument checks, the launch and (split vocabulary) the merge of the per-split statistics
template <Epi EPI, bool ENT = false>
static int forward(const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride, const void *weight,
                   int32_t V, int64_t weight_row_stride, const int64_t *labels, void *out, int out_dtype,
                   float *stat_max, float *stat_logsum, float *partial, int64_t partial_floats, int mode,
                   int32_t *status, const GradParams &gp, void *stream, const char *who, float *entropy = nullptr) {
  AA_REQUIRE(n_rows >= 0 && H > 0 && V > 0, AA_ERR_ARG, "%s: bad sizes", who);
  if (n_rows == 0) return AA_OK;
  AA_REQUIRE(hidden && weight && labels && out, AA_ERR_ARG, "%s: null pointer", who);
  AA_REQUIRE(H % BK == 0, AA_ERR_UNSUPPORTED, "%s: H=%d must be a multiple of %d", who, H, BK);
  AA_REQUIRE((reinterpret_cast<uintptr_t>(hidden) & 15) == 0 && (reinterpret_cast<uintptr_t>(weight) & 15) == 0 &&
                 hidden_row_stride % 8 == 0 && weight_row_stride % 8 == 0 && hidden_row_stride >= H && weight_row_stride >= H,
             AA_ERR_ALIGN, "%s: operands must be 16-byte aligned with 16-byte row strides", who);
  AA_REQUIRE(out_dtype == AA_BF16 || out_dtype == AA_F32, AA_ERR_DTYPE, "%s: out must be bf16 or f32", who);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "%s: bad mode", who);
  AA_REQUIRE(n_rows < (int64_t(1) << 31) - BM, AA_ERR_UNSUPPORTED, "%s: too many rows", who);
  const Schedule sc = make_schedule(n_rows, V, partial != nullptr, partial_floats, ENT ? 4 : 3);
  Params p{labels, n_rows, V, H, out, out_dtype, stat_max, stat_logsum, mode == AA_MODE_FAITHFUL ? 1 : 0, status,
           1, 1, 1, 1, 1, 1, partial, entropy};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = launch<EPI, ENT>(hidden, n_rows, H, hidden_row_stride, weight, V, weight_row_stride, p, gp, sc, st, who);
  p.v_splits = static_cast<int>(sc.splits);  // the merge kernel reads the split count
  const int64_t splits = sc.splits;
  if (rc || splits == 1) return rc;
  linear_logprob_merge_kernel<ENT><<<static_cast<unsigned>((n_rows + 255) / 256), 256, 0, st>>>(p);
  return check_launch(EPI == Epi::Logits ? "aa_linear_logits(merge)" : "aa_linear_logprob_fwd(merge)");
}
}  // namespace k6
}  // namespace aa

using namespace aa;

extern "C" int aa_linear_logprob_fwd(const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride,
                                     const void *weight, int32_t V, int64_t weight_row_stride, const int64_t *labels,
                                     void *out, int out_dtype, float *stat_max, float *stat_logsum, float *partial,
                                     int64_t partial_floats, int mode, int32_t *status, void *stream) {
  return k6::forward<k6::Epi::Lse>(hidden, n_rows, H, hidden_row_stride, weight, V, weight_row_stride, labels, out,
                                   out_dtype, stat_max, stat_logsum, partial, partial_floats, mode, status,
                                   k6::GradParams{nullptr, AA_F32, nullptr, 0, nullptr, AA_F32}, stream, "aa_linear_logprob_fwd");
}

extern "C" int aa_linear_logprob_fwd_entropy(const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride,
                                             const void *weight, int32_t V, int64_t weight_row_stride,
                                             const int64_t *labels, void *out, int out_dtype, float *stat_max,
                                             float *stat_logsum, float *partial, int64_t partial_floats, int mode,
                                             int32_t *status, float *entropy, void *stream) {
  AA_REQUIRE(n_rows == 0 || entropy, AA_ERR_ARG, "aa_linear_logprob_fwd_entropy: null entropy");
  return k6::forward<k6::Epi::Lse, true>(hidden, n_rows, H, hidden_row_stride, weight, V, weight_row_stride, labels, out,
                                         out_dtype, stat_max, stat_logsum, partial, partial_floats, mode, status,
                                         k6::GradParams{nullptr, AA_F32, nullptr, 0, nullptr, AA_F32}, stream,
                                         "aa_linear_logprob_fwd_entropy", entropy);
}

extern "C" int aa_linear_logits(const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride,
                                const void *weight, int32_t V, int64_t weight_row_stride, const int64_t *labels,
                                void *out, int out_dtype, float *stat_max, float *stat_logsum, float *partial,
                                int64_t partial_floats, int mode, int32_t *status, void *logits, int64_t ld,
                                void *stream) {
  if (n_rows > 0) {
    AA_REQUIRE(logits, AA_ERR_ARG, "aa_linear_logits: null pointer");
    const int64_t all_tiles = (static_cast<int64_t>(V) + k6::BN - 1) / k6::BN;
    AA_REQUIRE(V > 0 && ld >= all_tiles * k6::BN && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0,
               AA_ERR_ALIGN, "aa_linear_logits: ld must be >= ceil(V / 256) * 256, a multiple of 8, buffer 16-byte aligned");
  }
  return k6::forward<k6::Epi::Logits>(hidden, n_rows, H, hidden_row_stride, weight, V, weight_row_stride, labels, out,
                                      out_dtype, stat_max, stat_logsum, partial, partial_floats, mode, status,
                                      k6::GradParams{nullptr, AA_F32, static_cast<__nv_bfloat16 *>(logits), ld, nullptr, AA_F32}, stream,
                                      "aa_linear_logits");
}

// aa_linear_dlogits{,_entropy}: entropy == nullptr runs the plain kernel
static int linear_dlogits(const char *who, const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride,
                          const void *weight, int32_t V, int64_t weight_row_stride, const int64_t *labels,
                          const float *stat_max, const float *stat_logsum, const void *grad_rows, int grad_rows_dtype,
                          const float *entropy, const void *grad_entropy, int grad_entropy_dtype, void *dlogits,
                          int64_t ld, int mode, void *stream) {
  AA_REQUIRE(n_rows >= 0 && H > 0 && V > 0, AA_ERR_ARG, "%s: bad sizes", who);
  if (n_rows == 0) return AA_OK;
  AA_REQUIRE(hidden && weight && labels && stat_max && stat_logsum && grad_rows && dlogits, AA_ERR_ARG,
             "%s: null pointer", who);
  AA_REQUIRE(H % k6::BK == 0, AA_ERR_UNSUPPORTED, "%s: H=%d must be a multiple of %d", who, H, k6::BK);
  const int all_tiles = (V + k6::BN - 1) / k6::BN;
  AA_REQUIRE(ld >= static_cast<int64_t>(all_tiles) * k6::BN && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(dlogits) & 15) == 0,
             AA_ERR_ALIGN, "%s: ld must be >= ceil(V / 256) * 256, a multiple of 8, buffer 16-byte aligned", who);
  AA_REQUIRE((reinterpret_cast<uintptr_t>(hidden) & 15) == 0 && (reinterpret_cast<uintptr_t>(weight) & 15) == 0 &&
                 hidden_row_stride % 8 == 0 && weight_row_stride % 8 == 0 && hidden_row_stride >= H && weight_row_stride >= H,
             AA_ERR_ALIGN, "%s: operands must be 16-byte aligned with 16-byte row strides", who);
  AA_REQUIRE(grad_rows_dtype == AA_BF16 || grad_rows_dtype == AA_F16 || grad_rows_dtype == AA_F32, AA_ERR_DTYPE,
             "%s: bad grad dtype", who);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "%s: bad mode", who);
  AA_REQUIRE(n_rows < (int64_t(1) << 31) - k6::BM, AA_ERR_UNSUPPORTED, "%s: too many rows", who);
  const k6::Schedule sc = k6::make_schedule(n_rows, V, true, -1);
  k6::Params p{labels, n_rows, V, H, nullptr, AA_BF16, const_cast<float *>(stat_max), const_cast<float *>(stat_logsum),
               mode == AA_MODE_FAITHFUL ? 1 : 0, nullptr, 1, 1, 1, 1, 1, 1, nullptr, const_cast<float *>(entropy)};
  k6::GradParams gp{grad_rows, grad_rows_dtype, static_cast<__nv_bfloat16 *>(dlogits), ld, grad_entropy,
                    grad_entropy_dtype};
  if (entropy)
    return k6::launch<k6::Epi::DLogits, true>(hidden, n_rows, H, hidden_row_stride, weight, V, weight_row_stride, p, gp,
                                              sc, static_cast<cudaStream_t>(stream), who);
  return k6::launch<k6::Epi::DLogits>(hidden, n_rows, H, hidden_row_stride, weight, V, weight_row_stride, p, gp, sc,
                          static_cast<cudaStream_t>(stream), who);
}

extern "C" int aa_linear_dlogits(const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride,
                                 const void *weight, int32_t V, int64_t weight_row_stride, const int64_t *labels,
                                 const float *stat_max, const float *stat_logsum, const void *grad_rows,
                                 int grad_rows_dtype, void *dlogits, int64_t ld, int mode, void *stream) {
  return linear_dlogits("aa_linear_dlogits", hidden, n_rows, H, hidden_row_stride, weight, V, weight_row_stride, labels,
                        stat_max, stat_logsum, grad_rows, grad_rows_dtype, nullptr, nullptr, AA_F32, dlogits, ld, mode,
                        stream);
}

extern "C" int aa_linear_dlogits_entropy(const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride,
                                         const void *weight, int32_t V, int64_t weight_row_stride, const int64_t *labels,
                                         const float *stat_max, const float *stat_logsum, const void *grad_rows,
                                         int grad_rows_dtype, const float *entropy, const void *grad_entropy,
                                         int grad_entropy_dtype, void *dlogits, int64_t ld, int mode, void *stream) {
  AA_REQUIRE(n_rows == 0 || (entropy && grad_entropy), AA_ERR_ARG,
             "aa_linear_dlogits_entropy: entropy and grad_entropy are required");
  AA_REQUIRE(grad_entropy_dtype == AA_BF16 || grad_entropy_dtype == AA_F16 || grad_entropy_dtype == AA_F32, AA_ERR_DTYPE,
             "aa_linear_dlogits_entropy: bad grad_entropy dtype");
  return linear_dlogits("aa_linear_dlogits_entropy", hidden, n_rows, H, hidden_row_stride, weight, V, weight_row_stride,
                        labels, stat_max, stat_logsum, grad_rows, grad_rows_dtype, n_rows ? entropy : nullptr,
                        grad_entropy, grad_entropy_dtype, dlogits, ld, mode, stream);
}
