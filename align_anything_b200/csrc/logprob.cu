// logprob.cu -- K1 / K1b: per-token log-prob (row log-softmax over V fused with the label
// gather) and its backward, for ragged row lists over non-contiguous logits views.
//
// Replaces utils/tools.py:402-413 (gather_log_probabilities) + autograd of F.log_softmax /
// torch.gather, and the per-sample slicing loops around them (trainers/text_to_text/dpo.py:133-142,
// trainers/text_image_to_text/ppo.py:229-239).  The (rows, V) log-prob tile is never written.
//
// HBM-bound streaming reduction: one CTA owns one row at a time (persistent, grid-strided);
// 128-bit streaming loads over the 16-byte-aligned body of the row, scalar peel for the
// (<8 element) head / tail when the row start is only 2-byte aligned (odd V such as 128257);
// per-thread online softmax in the exp2 domain, warp-shuffle + shared-memory merge of the
// (max, sum) partials.
#include <atomic>

#include "common.cuh"
#include "logprob_math.cuh"

namespace aa {

struct FwdParams {
  const void *logits;
  int64_t row_stride;
  int V;
  const int64_t *labels;
  int64_t ignore_index;  // rows whose label equals this are skipped (out = 0) when use_ignore != 0
  int use_ignore;
  RowMap map;
  int64_t n_rows;
  void *out;
  int out_dtype;
  float *stat_max;
  float *stat_logsum;
  int32_t *status;
  float log2e;  // = kLog2e, passed at run time so that ptxas keeps the packed FMUL2 (no immediate form)
  // entropy kernels only (ENT = true): fp32 entropy of the row at its out position, for out positions < n_entropy
  float *entropy;
  int64_t n_entropy;
};

struct BwdParams {
  const void *logits;
  int64_t row_stride;
  int V;
  const int64_t *labels;
  int64_t ignore_index;
  int use_ignore;
  RowMap map;
  int64_t n_rows;
  const int64_t *seg_tile_row;
  const float *stat_max;
  const float *stat_logsum;
  const void *grad_rows;
  int grad_rows_dtype;
  const float *grad_seg;
  const void *grad_scale;  // optional device scalar (dtype grad_scale_dtype): the upstream d loss of a fused loss node
  int grad_scale_dtype;
  void *grad_logits;
  int64_t grad_row_stride;
  int64_t n_tile_rows;
  float zero;  // +0.0f supplied at run time (see f2_round_bf16 in common.cuh)
  const int64_t *extra_zero_rows;  // n_tile_rows == 0 only: tile rows to zero-fill after the scored rows
  int64_t n_extra;
  // entropy-gradient kernels only (ENT = true): the forward's fp32 entropy and its upstream gradient, both indexed like
  // grad_rows (grad_entropy in dtype grad_entropy_dtype); grad_scale multiplies g_H as it multiplies g
  const float *entropy;
  const void *grad_entropy;
  int grad_entropy_dtype;
};
__host__ __device__ __forceinline__ int64_t bwd_work_rows(const BwdParams &p) {
  return p.n_tile_rows > 0 ? p.n_tile_rows : p.n_rows + p.n_extra;
}

// ---- K1 forward, LDG: direct vectorised loads (rows of 128 KB and more, see launch_fwd) -------------
template <typename T, int THREADS, int UNROLL, bool ENT = false>
__global__ void __launch_bounds__(THREADS) logprob_fwd_kernel(const FwdParams p) {
  constexpr int E = Traits<T>::kVec;
  __shared__ float sh_m[32], sh_s[32];
  __shared__ float sh_t[ENT ? 32 : 1];
  const int tid = threadIdx.x;
  const T *__restrict__ logits = reinterpret_cast<const T *>(p.logits);
  const int V = p.V;
  const f32x2 L2 = f2_splat(p.log2e);

  // p.n_rows is an upper bound when the plan was built on the device (aa_tail_plan_build: the response lengths never
  // visit the host); the table's last prefix entry is the exact count
  const int64_t n_rows = min(p.n_rows, __ldg(p.map.seg_cum + p.map.n_seg));
  for (int64_t row = blockIdx.x; row < n_rows; row += gridDim.x) {
    const int seg = upper_segment(p.map.seg_cum, p.map.n_seg, row);
    const int64_t j = row - __ldg(p.map.seg_cum + seg);
    const T *x = logits + __ldg(p.map.seg_logit_off + seg) + j * p.row_stride;

    const int64_t y = __ldg(p.labels + __ldg(p.map.seg_label_off + seg) + j);  // same address in every thread
    if (p.use_ignore && y == p.ignore_index) {  // ignored position (cross-entropy ignore_index): no traffic
      if (tid == 0) {
        store_from_float(p.out, __ldg(p.map.seg_out_off + seg) + j, p.out_dtype, 0.f);
        if constexpr (ENT) {
          const int64_t o = __ldg(p.map.seg_out_off + seg) + j;
          if (o < p.n_entropy) p.entropy[o] = 0.f;
        }
        if (p.stat_max) {
          p.stat_max[row] = 0.f;
          p.stat_logsum[row] = 0.f;
        }
      }
      continue;
    }
    float xy = 0.f;
    bool y_ok = true;
    if (tid == 0) {  // label column: one 2/4-byte load, issued before the streaming loop
      y_ok = (y >= 0) && (y < V);
      xy = y_ok ? Traits<T>::to_float(x[y]) : NAN;
    }

    const int mis = static_cast<int>((reinterpret_cast<uintptr_t>(x) & 15) / sizeof(T));
    const int head = mis ? min(E - mis, V) : 0;
    const int nvec = (V - head) / E;
    const int tail0 = head + nvec * E;
    const uint4 *body = reinterpret_cast<const uint4 *>(x + head);

    float m = -INFINITY, s = 0.f, t = 0.f;
    if (tid < head) lse_push_t<ENT>(m, s, t, Traits<T>::to_float(x[tid]));
    if (tid < V - tail0) lse_push_t<ENT>(m, s, t, Traits<T>::to_float(x[tail0 + tid]));

    int k = tid;
    for (; k + (UNROLL - 1) * THREADS < nvec; k += UNROLL * THREADS) {
      uint4 v[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) v[u] = ldg_stream(body + k + u * THREADS);
      fold_batch_t<T, UNROLL, ENT>(v, m, s, t, L2);
    }
    if (k < nvec) {  // last, partial batch: missing vectors are replaced by -inf (exp -> 0), one fold instead of
                     // up to UNROLL-1 single-vector folds (each of which pays its own max / rescale)
      uint4 v[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u)
        v[u] = (k + u * THREADS < nvec) ? ldg_stream(body + k + u * THREADS) : bulk::neg_inf_vec<T>();
      fold_batch_t<T, UNROLL, ENT>(v, m, s, t, L2);
    }

    block_lse_t<THREADS, ENT>(m, s, t, sh_m, sh_s, sh_t);
    if (tid == 0) {
      const float logsum = logf(s);
      float lp = (xy - m) - logsum;  // same association as ATen's `x - max - log(sum)`
      if (!y_ok) {
        lp = NAN;
        if (p.status) atomicOr(p.status, AA_STATUS_LABEL_OOB);
      }
      store_from_float(p.out, __ldg(p.map.seg_out_off + seg) + j, p.out_dtype, lp);
      if constexpr (ENT) {
        const int64_t o = __ldg(p.map.seg_out_off + seg) + j;
        if (o < p.n_entropy) p.entropy[o] = entropy_of(logsum, s, t);
      }
      if (p.stat_max) {
        p.stat_max[row] = m;
        p.stat_logsum[row] = logsum;
      }
    }
    __syncthreads();  // sh_m / sh_s reuse
  }
}

// ---- K1 forward, default: rows streamed through a cp.async.bulk ring ---------------------------------
// One producer lane walks the CTA's rows and owns everything that needs a dependent global load: segment
// lookup, logits pointer, label, ignore_index test.  Ignored rows it writes itself (output 0, no traffic);
// for every other row it hands a descriptor to the consumers through a small shared-memory queue and
// streams the row's 16-byte-aligned body into a ring of shared-memory stages with cp.async.bulk (SASS:
// UBLKCP), completion signalled on mbarriers.  The ring runs across row boundaries, so the copy engine is
// already fetching the next row while the consumers reduce the current one.  Eight consumer warps read the
// stages with conflict-free LDS.128 and run the online softmax of the LDG kernel above.  The label logit is
// picked out of the staged chunk that holds it; only the (< 8 element) head / tail of an odd-V row and a
// label outside the aligned body are scalar loads, issued at row start and consumed at row end.  The
// row-end merge costs one named barrier over the consumers (the (m, s) scratch is double-buffered).
// Tensor maps are not needed (and could not describe V = 128257 anyway: a TMA tensor map wants 16-byte
// row strides); the 1-D bulk copy only needs the 16-byte-aligned body that the head / tail peel isolates.
struct __align__(16) FwdRowDesc {
  const void *x;    // logits row; nullptr: no more rows for this CTA
  int64_t out_idx;  // element index in p.out
  int64_t row;      // flat row index (p.stat_max / p.stat_logsum)
  int32_t y;        // label column, -1 when out of range
};
constexpr int kFwdDescs = 8;  // descriptor queue depth (rows the producer may run ahead of the consumers)

template <int CONSUMERS, int STAGES, int UNROLL>
constexpr size_t fwd_ring_smem() {
  return static_cast<size_t>(STAGES) * CONSUMERS * UNROLL * 16 + 2 * STAGES * sizeof(uint64_t) +
         2 * kFwdDescs * sizeof(uint64_t) + kFwdDescs * sizeof(FwdRowDesc);
}

template <typename T, int CONSUMERS, int STAGES, int UNROLL, bool ENT = false>
__global__ void __launch_bounds__(CONSUMERS + 32) logprob_fwd_ring_kernel(const FwdParams p) {
  constexpr int E = Traits<T>::kVec;
  constexpr int NW = CONSUMERS / kWarp;
  constexpr int STAGE_VECS = CONSUMERS * UNROLL;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint4 *ring = reinterpret_cast<uint4 *>(smem_raw);
  uint64_t *full = reinterpret_cast<uint64_t *>(smem_raw + static_cast<size_t>(STAGES) * STAGE_VECS * 16);
  uint64_t *empty = full + STAGES;
  uint64_t *dfull = empty + STAGES;
  uint64_t *dempty = dfull + kFwdDescs;
  FwdRowDesc *desc = reinterpret_cast<FwdRowDesc *>(dempty + kFwdDescs);
  __shared__ float sh_m[2][NW], sh_s[2][NW], sh_xy[2];
  __shared__ float sh_t[2][ENT ? NW : 1];
  const int tid = threadIdx.x;
  const int V = p.V;
  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) {
      bulk::mbar_init(full + i, 1);
      bulk::mbar_init(empty + i, NW);
    }
    for (int i = 0; i < kFwdDescs; ++i) {
      bulk::mbar_init(dfull + i, 1);
      bulk::mbar_init(dempty + i, NW);
    }
    bulk::fence_barrier_init();
  }
  __syncthreads();
  int stage = 0, dq = 0;
  uint32_t phase = 0, dphase = 0;

  if (tid >= CONSUMERS) {
    // ---------------- producer warp: one elected lane ----------------
    if (tid != CONSUMERS) return;
    const T *__restrict__ logits = reinterpret_cast<const T *>(p.logits);
    // p.n_rows is an upper bound when the plan was built on the device: see the LDG kernel
    const int64_t n_rows = min(p.n_rows, __ldg(p.map.seg_cum + p.map.n_seg));
    int64_t seg_lo = 0, seg_hi = 0, logit_off = 0, label_off = 0, out_off = 0;
    for (int64_t row = blockIdx.x; row < n_rows; row += gridDim.x) {
      if (row >= seg_hi) {  // rows only move forward: search the plan on a segment change only
        const int seg = upper_segment(p.map.seg_cum, p.map.n_seg, row);
        seg_lo = __ldg(p.map.seg_cum + seg);
        seg_hi = __ldg(p.map.seg_cum + seg + 1);
        logit_off = __ldg(p.map.seg_logit_off + seg);
        label_off = __ldg(p.map.seg_label_off + seg);
        out_off = __ldg(p.map.seg_out_off + seg);
      }
      const int64_t j = row - seg_lo;
      const int64_t y = __ldg(p.labels + label_off + j);
      if (p.use_ignore && y == p.ignore_index) {  // ignored position (cross-entropy ignore_index): no traffic
        store_from_float(p.out, out_off + j, p.out_dtype, 0.f);
        if constexpr (ENT) {
          if (out_off + j < p.n_entropy) p.entropy[out_off + j] = 0.f;
        }
        if (p.stat_max) {
          p.stat_max[row] = 0.f;
          p.stat_logsum[row] = 0.f;
        }
        continue;
      }
      const T *x = logits + logit_off + j * p.row_stride;
      bulk::mbar_wait(dempty + dq, dphase ^ 1u);
      desc[dq] = FwdRowDesc{x, out_off + j, row, (y >= 0 && y < V) ? static_cast<int32_t>(y) : -1};
      bulk::mbar_arrive(dfull + dq);
      if (++dq == kFwdDescs) {
        dq = 0;
        dphase ^= 1u;
      }
      const int mis = static_cast<int>((reinterpret_cast<uintptr_t>(x) & 15) / sizeof(T));
      const int head = mis ? min(E - mis, V) : 0;
      const int nvec = (V - head) / E;
      const uint4 *body = reinterpret_cast<const uint4 *>(x + head);
      for (int v0 = 0; v0 < nvec; v0 += STAGE_VECS) {
        const uint32_t bytes = static_cast<uint32_t>(min(STAGE_VECS, nvec - v0)) * 16u;
        bulk::mbar_wait(empty + stage, phase ^ 1u);
        bulk::mbar_expect_tx(full + stage, bytes);
        bulk::bulk_g2s(ring + static_cast<size_t>(stage) * STAGE_VECS, body + v0, bytes, full + stage);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }
    }
    bulk::mbar_wait(dempty + dq, dphase ^ 1u);
    desc[dq].x = nullptr;
    bulk::mbar_arrive(dfull + dq);
    return;
  }

  // ---------------- consumer warps ----------------
  const f32x2 L2 = f2_splat(p.log2e);
  const int lane = tid & 31, wid = tid >> 5;
  for (int par = 0;; par ^= 1) {
    bulk::mbar_wait(dfull + dq, dphase);
    const FwdRowDesc d = desc[dq];
    __syncwarp();
    if (lane == 0) bulk::mbar_arrive(dempty + dq);
    if (++dq == kFwdDescs) {
      dq = 0;
      dphase ^= 1u;
    }
    if (d.x == nullptr) break;
    const T *x = reinterpret_cast<const T *>(d.x);
    const int mis = static_cast<int>((reinterpret_cast<uintptr_t>(x) & 15) / sizeof(T));
    const int head = mis ? min(E - mis, V) : 0;
    const int nvec = (V - head) / E;
    const int tail0 = head + nvec * E;
    const int yb = (d.y >= head && d.y < tail0) ? d.y - head : -1;  // label offset in the aligned body
    const int yv = yb >= 0 ? yb / E : -1;
    // scalar loads: issued now, consumed after the body has streamed by
    const float hx = tid < head ? Traits<T>::to_float(x[tid]) : -INFINITY;
    const float tx = tid < V - tail0 ? Traits<T>::to_float(x[tail0 + tid]) : -INFINITY;
    const float xy_peel = (tid == 0 && d.y >= 0 && yb < 0) ? Traits<T>::to_float(x[d.y]) : 0.f;

    float m = -INFINITY, s = 0.f, t = 0.f;
    for (int v0 = 0; v0 < nvec; v0 += STAGE_VECS) {
      const int n = min(STAGE_VECS, nvec - v0);
      bulk::mbar_wait(full + stage, phase);
      const uint4 *buf = ring + static_cast<size_t>(stage) * STAGE_VECS;
      uint4 v[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const int k = tid + u * CONSUMERS;
        v[u] = (k < n) ? buf[k] : bulk::neg_inf_vec<T>();
        if (v0 + k == yv) {  // the label column lies in this vector
          const int e = yb - yv * E;
          float lo, hi;
          if constexpr (sizeof(T) == 4) {
            lo = hi = __uint_as_float(get_word(v[u], e));
          } else {
            unpack2<T>(get_word(v[u], e >> 1), lo, hi);
          }
          sh_xy[par] = (e & 1) ? hi : lo;
        }
      }
      // order this warp's generic-proxy reads of the stage before the copy engine's next write to it
      // (compute-sanitizer racecheck reports the WAR pair without the proxy fence)
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) bulk::mbar_arrive(empty + stage);  // this warp's reads of the stage are done
      fold_batch_t<T, UNROLL, ENT>(v, m, s, t, L2);
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1u;
      }
    }
    lse_push_t<ENT>(m, s, t, hx);
    lse_push_t<ENT>(m, s, t, tx);

    // merge the partials of the CONSUMERS threads.  Named barrier 1 leaves the producer out; the scratch is
    // double-buffered by row parity, so warp 0 reading this row's partials cannot race the next row's writes
    // (those come after the next row's barrier, which warp 0 reaches only when it is done here).
    warp_lse_t<ENT>(m, s, t);
    if (lane == 0) {
      sh_m[par][wid] = m;
      sh_s[par][wid] = s;
      if constexpr (ENT) sh_t[par][wid] = t;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
    if (wid == 0) {
      m = lane < NW ? sh_m[par][lane] : -INFINITY;
      s = lane < NW ? sh_s[par][lane] : 0.f;
      if constexpr (ENT) t = lane < NW ? sh_t[par][lane] : 0.f;
      warp_lse_t<ENT>(m, s, t);
      if (tid == 0) {
        const float logsum = logf(s);
        const float xy = yb >= 0 ? sh_xy[par] : xy_peel;
        float lp = (xy - m) - logsum;  // same association as ATen's `x - max - log(sum)`
        if (d.y < 0) {
          lp = NAN;
          if (p.status) atomicOr(p.status, AA_STATUS_LABEL_OOB);
        }
        store_from_float(p.out, d.out_idx, p.out_dtype, lp);
        if constexpr (ENT) {
          if (d.out_idx < p.n_entropy) p.entropy[d.out_idx] = entropy_of(logsum, s, t);
        }
        if (p.stat_max) {
          p.stat_max[d.row] = m;
          p.stat_logsum[d.row] = logsum;
        }
      }
    }
  }
}

// ---- K1b backward -------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void zero_row(T *g, int V) {
  constexpr int E = Traits<T>::kVec;
  const int mis = static_cast<int>((reinterpret_cast<uintptr_t>(g) & 15) / sizeof(T));
  const int head = mis ? min(E - mis, V) : 0;
  const int nvec = (V - head) / E;
  const int tail0 = head + nvec * E;
  const int tid = threadIdx.x;
  if (tid < head) g[tid] = Traits<T>::from_float(0.f);
  if (tid < V - tail0) g[tail0 + tid] = Traits<T>::from_float(0.f);
  uint4 *body = reinterpret_cast<uint4 *>(g + head);
  const uint4 z = make_uint4(0, 0, 0, 0);
  for (int k = tid; k < nvec; k += blockDim.x) stg_stream(body + k, z);
}

template <typename T, int THREADS, int UNROLL, bool FAITHFUL>
__global__ void __launch_bounds__(THREADS) logprob_bwd_kernel(const BwdParams p) {
  constexpr int E = Traits<T>::kVec;
  const int tid = threadIdx.x;
  const int V = p.V;
  const T *__restrict__ logits = reinterpret_cast<const T *>(p.logits);
  T *__restrict__ grad = reinterpret_cast<T *>(p.grad_logits);
  const bool tile_mode = p.n_tile_rows > 0;
  const int64_t n_work = bwd_work_rows(p);

  for (int64_t work = blockIdx.x; work < n_work; work += gridDim.x) {
    int seg;
    int64_t j;
    T *g_out;
    if (!tile_mode && work >= p.n_rows) {  // listed zero rows
      zero_row<T>(grad + __ldg(p.extra_zero_rows + (work - p.n_rows)) * p.grad_row_stride, V);
      continue;
    }
    if (tile_mode) {
      g_out = grad + work * p.grad_row_stride;
      bool scored = false;
      seg = 0;
      j = 0;
      if (p.map.n_seg > 0 && work >= __ldg(p.seg_tile_row)) {
        seg = upper_segment(p.seg_tile_row, p.map.n_seg, work);
        j = work - __ldg(p.seg_tile_row + seg);
        scored = j < (__ldg(p.map.seg_cum + seg + 1) - __ldg(p.map.seg_cum + seg));
      }
      if (!scored) {
        zero_row<T>(g_out, V);
        continue;
      }
    } else {
      seg = upper_segment(p.map.seg_cum, p.map.n_seg, work);
      j = work - __ldg(p.map.seg_cum + seg);
      g_out = grad + (__ldg(p.seg_tile_row + seg) + j) * p.grad_row_stride;
    }
    const int64_t flat = __ldg(p.map.seg_cum + seg) + j;
    const T *x = logits + __ldg(p.map.seg_logit_off + seg) + j * p.row_stride;

    float g = 1.f;
    if (p.grad_rows) g *= load_as_float(p.grad_rows, __ldg(p.map.seg_out_off + seg) + j, p.grad_rows_dtype);
    if (p.grad_seg) g *= __ldg(p.grad_seg + seg);
    if (p.grad_scale) g *= load_as_float(p.grad_scale, 0, p.grad_scale_dtype);
    if (p.use_ignore && __ldg(p.labels + __ldg(p.map.seg_label_off + seg) + j) == p.ignore_index) g = 0.f;
    if (g == 0.f) {  // masked / prompt / ignored rows: 0 * softmax, no need to read the row
      zero_row<T>(g_out, V);
      continue;
    }
    const float m = __ldg(p.stat_max + flat);
    const float logsum = __ldg(p.stat_logsum + flat);
    const float lse = m + logsum;
    const float c_f32 = -lse * kLog2e;
    // F32 mode: p_j = 2^(x_j*log2e + c_f32) * 2^(residual of the rounded offset), folded into -g
    const float neg_g = FAITHFUL ? -g : -g * ex2_approx(fmaf(-lse, kLog2e, -c_f32));
    const GradConsts gk = make_grad_consts(m, logsum, c_f32, neg_g, p.zero);

    const bool same_phase =
        ((reinterpret_cast<uintptr_t>(x) ^ reinterpret_cast<uintptr_t>(g_out)) & 15) == 0;
    if (same_phase) {
      const int mis = static_cast<int>((reinterpret_cast<uintptr_t>(x) & 15) / sizeof(T));
      const int head = mis ? min(E - mis, V) : 0;
      const int nvec = (V - head) / E;
      const int tail0 = head + nvec * E;
      if (tid < head)
        g_out[tid] = Traits<T>::from_float(
            neg_g * prob_of<T, FAITHFUL>(Traits<T>::to_float(x[tid]), m, logsum, c_f32));
      if (tid < V - tail0)
        g_out[tail0 + tid] = Traits<T>::from_float(
            neg_g * prob_of<T, FAITHFUL>(Traits<T>::to_float(x[tail0 + tid]), m, logsum, c_f32));
      const uint4 *src = reinterpret_cast<const uint4 *>(x + head);
      uint4 *dst = reinterpret_cast<uint4 *>(g_out + head);
      int k = tid;
      for (; k + (UNROLL - 1) * THREADS < nvec; k += UNROLL * THREADS) {
        uint4 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) v[u] = ldg_stream(src + k + u * THREADS);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u)
          stg_stream(dst + k + u * THREADS, vec_grad<T, FAITHFUL>(v[u], gk));
      }
      for (; k < nvec; k += THREADS)
        stg_stream(dst + k, vec_grad<T, FAITHFUL>(ldg_stream(src + k), gk));
    } else {
      // logits view and gradient tile disagree on the 16-byte phase of this row: element loop
      for (int c = tid; c < V; c += THREADS)
        g_out[c] = Traits<T>::from_float(
            neg_g * prob_of<T, FAITHFUL>(Traits<T>::to_float(x[c]), m, logsum, c_f32));
    }
    // the label column: grad = g - p_y * g (ATen: grad_out - exp(out) * sum(grad_out))
    __syncthreads();
    if (tid == 0) {
      const int64_t y = __ldg(p.labels + __ldg(p.map.seg_label_off + seg) + j);
      if (y >= 0 && y < V) {
        const float py = prob_of<T, FAITHFUL>(Traits<T>::to_float(x[y]), m, logsum, c_f32);
        g_out[y] = Traits<T>::from_float(FAITHFUL ? __fsub_rn(g, __fmul_rn(py, g)) : fmaf(py, neg_g, g));
      }
    }
  }
}

// ---- K1b, TMA-staged (default whenever row_scratch is given) -------------------------------------
// The backward needs no per-row reduction (max / logsum come from the forward).  A tiny prep kernel
// resolves each row once (segment search, label, saved stats, upstream gradient) into a 32-byte record,
// so the TMA kernel below reads one record per row instead of searching the row plan.
struct __align__(16) RowRec {
  int64_t x_off;   // element offset of the logits row
  int64_t g_row;   // row index in the gradient tile
  float m, logsum, g;
  int32_t y;       // label column; -1: out of range (no one-hot term); -2: zero-fill the row
};
// the entropy-gradient kernels' record: RowRec, then the row's entropy and its upstream gradient
struct __align__(16) RowRecEnt {
  RowRec r;
  float H, gH;
  int32_t pad[2];
};
static_assert(sizeof(RowRec) == 32 && sizeof(RowRecEnt) == 48, "records are read as 16-byte vectors");

template <bool ENT = false>
__global__ void bwd_row_prep_kernel(const BwdParams p, RowRec *__restrict__ rec) {
  const bool tile_mode = p.n_tile_rows > 0;
  const int64_t n_work = bwd_work_rows(p);
  const int64_t work = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (work >= n_work) return;
  RowRec r;
  r.x_off = 0; r.g_row = work; r.m = 0.f; r.logsum = 0.f; r.g = 0.f; r.y = -2;
  int seg = 0;
  int64_t j = 0;
  bool scored;
  int64_t slot = work;  // where the record goes in the work list
  if (!tile_mode && work >= p.n_rows) {  // listed zero rows come after the scored rows: balanced static stride
    r.g_row = __ldg(p.extra_zero_rows + (work - p.n_rows));
    scored = false;
  } else if (tile_mode) {
    // every tile row is work (the row layout is only known on the device).  The work list is ORDERED: the scored rows
    // first, in flat row order, then the zero rows -- the persistent kernel's static stride then sees equally expensive
    // rows next to each other (rows in tile order gave +-40% scored rows per CTA in the PPO shape)
    scored = false;
    int64_t scored_before = 0;
    if (p.map.n_seg > 0 && work >= __ldg(p.seg_tile_row)) {
      seg = upper_segment(p.seg_tile_row, p.map.n_seg, work);
      j = work - __ldg(p.seg_tile_row + seg);
      const int64_t first = __ldg(p.map.seg_cum + seg), cnt = __ldg(p.map.seg_cum + seg + 1) - first;
      scored = j < cnt;
      scored_before = first + min(j, cnt);
    }
    const int64_t total_scored = __ldg(p.map.seg_cum + p.map.n_seg);
    slot = scored ? scored_before : total_scored + (work - scored_before);
  } else {
    seg = upper_segment(p.map.seg_cum, p.map.n_seg, work);
    j = work - __ldg(p.map.seg_cum + seg);
    r.g_row = __ldg(p.seg_tile_row + seg) + j;
    scored = true;
  }
  float H = 0.f, gH = 0.f;
  if (scored) {
    const int64_t flat = __ldg(p.map.seg_cum + seg) + j;
    float g = 1.f;
    if (p.grad_rows) g *= load_as_float(p.grad_rows, __ldg(p.map.seg_out_off + seg) + j, p.grad_rows_dtype);
    if (p.grad_seg) g *= __ldg(p.grad_seg + seg);
    if (p.grad_scale) g *= load_as_float(p.grad_scale, 0, p.grad_scale_dtype);
    if constexpr (ENT) {
      const int64_t o = __ldg(p.map.seg_out_off + seg) + j;
      gH = load_as_float(p.grad_entropy, o, p.grad_entropy_dtype);
      if (p.grad_scale) gH *= load_as_float(p.grad_scale, 0, p.grad_scale_dtype);
      H = __ldg(p.entropy + o);
    }
    const int64_t y = __ldg(p.labels + __ldg(p.map.seg_label_off + seg) + j);
    if (p.use_ignore && y == p.ignore_index) {
      g = 0.f;
      if constexpr (ENT) gH = 0.f;
    }
    if (g != 0.f || (ENT && gH != 0.f)) {  // g == 0 (masked / prompt / ignored rows): plain zero row
      r.x_off = __ldg(p.map.seg_logit_off + seg) + j * p.row_stride;
      r.m = __ldg(p.stat_max + flat);
      r.logsum = __ldg(p.stat_logsum + flat);
      r.g = g;
      r.y = (y >= 0 && y < p.V) ? static_cast<int32_t>(y) : -1;
    }
  }
  if constexpr (ENT)
    reinterpret_cast<RowRecEnt *>(rec)[slot] = RowRecEnt{r, H, gH, {0, 0}};
  else
    rec[slot] = r;
}

// A pure copy with the one-CTA-per-row access structure of the LDG kernel above stays below what the copy
// engine (cp.async.bulk global->smem, smem->global, 64 KB in flight per SM) reaches, which is cudaMemcpy
// speed.  So the backward moves its data with the TMA engine in both directions and the SM only touches
// shared memory:
//   producer lane : RowRec -> cp.async.bulk loads of stage-sized chunks of the row's aligned body into a ring
//                   (full mbarriers, expect_tx), and -- lagging LAG chunks behind -- cp.async.bulk
//                   STORES of the chunks the consumers have finished (done mbarriers); zero rows are
//                   stored straight from a zeroed shared-memory buffer, no SM data path at all;
//   8 consumer warps: LDS.128 -> grad math (f32x2, Veltkamp rounding) -> STS.128 in place, one-hot label
//                   patched in registers, fence.proxy.async, arrive(done).
// Rows whose logits and gradient addresses disagree modulo 16 fall back to an element loop.
// ENT: the records are RowRecEnt and rows with g_H != 0 get the entropy correction (vec_grad_ent).
template <typename T, int CONSUMERS, int STAGES, int UNROLL, int LAG, bool FAITHFUL, bool ENT = false>
__global__ void __launch_bounds__(CONSUMERS + 32)
    logprob_bwd_tma_kernel(const T *__restrict__ logits, T *__restrict__ grad, int64_t grad_row_stride, int V,
                           const RowRec *__restrict__ rec, int64_t n_work, float zero) {
  constexpr int E = Traits<T>::kVec;
  constexpr int STAGE_VECS = CONSUMERS * UNROLL;
  constexpr int kRecVecs = (ENT ? sizeof(RowRecEnt) : sizeof(RowRec)) / 16;
  static_assert(LAG >= 1 && LAG < STAGES, "LAG must leave at least one free stage");
  extern __shared__ __align__(128) uint8_t smem_raw[];
  uint4 *ring = reinterpret_cast<uint4 *>(smem_raw);
  uint4 *zero_buf = ring + static_cast<size_t>(STAGES) * STAGE_VECS;
  uint64_t *full = reinterpret_cast<uint64_t *>(zero_buf + STAGE_VECS);
  uint64_t *done = full + STAGES;
  uint64_t *st_dst = done + STAGES;                             // destination of the chunk held by each stage
  uint32_t *st_bytes = reinterpret_cast<uint32_t *>(st_dst + STAGES);
  const int tid = threadIdx.x;
  for (int i = tid; i < STAGE_VECS; i += CONSUMERS + 32) zero_buf[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) {
      bulk::mbar_init(full + i, 1);
      bulk::mbar_init(done + i, CONSUMERS / kWarp);
    }
    bulk::fence_barrier_init();
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // zero_buf is read by the async proxy
  __syncthreads();

  if (tid >= CONSUMERS) {
    // ------------------------------ producer lane ------------------------------
    if (tid != CONSUMERS) return;
    int64_t it = 0;       // chunks loaded so far
    int64_t retired = 0;  // chunks stored so far
    auto retire_one = [&]() {
      const int s = static_cast<int>(retired % STAGES);
      bulk::mbar_wait(done + s, static_cast<uint32_t>((retired / STAGES) & 1));
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(st_dst[s]),
                   "r"(bulk::smem_u32(ring + static_cast<size_t>(s) * STAGE_VECS)), "r"(st_bytes[s])
                   : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      ++retired;
    };
    for (int64_t r = blockIdx.x; r < n_work; r += gridDim.x) {
      const int4 *rv = reinterpret_cast<const int4 *>(rec) + r * kRecVecs;
      const int4 r0 = __ldg(rv);
      const int4 r1 = __ldg(rv + 1);
      const int64_t x_off = (static_cast<int64_t>(static_cast<uint32_t>(r0.y)) << 32) | static_cast<uint32_t>(r0.x);
      const int64_t g_row = (static_cast<int64_t>(static_cast<uint32_t>(r0.w)) << 32) | static_cast<uint32_t>(r0.z);
      const int y = r1.w;
      T *g_out = grad + g_row * grad_row_stride;
      const int mis = static_cast<int>((reinterpret_cast<uintptr_t>(g_out) & 15) / sizeof(T));
      const int head = mis ? min(E - mis, V) : 0;
      const int nvec = (V - head) / E;
      const int tail0 = head + nvec * E;
      uint4 *gbody = reinterpret_cast<uint4 *>(g_out + head);
      if (y == -2) {  // zero row: the copy engine writes it from the zero buffer
        for (int e = 0; e < head; ++e) g_out[e] = Traits<T>::from_float(0.f);
        for (int e = tail0; e < V; ++e) g_out[e] = Traits<T>::from_float(0.f);
        for (int v0 = 0; v0 < nvec; v0 += STAGE_VECS) {
          const uint32_t bytes = static_cast<uint32_t>(min(STAGE_VECS, nvec - v0)) * 16u;
          asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gbody + v0),
                       "r"(bulk::smem_u32(zero_buf)), "r"(bytes)
                       : "memory");
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        continue;
      }
      const T *x = logits + x_off;
      if (((reinterpret_cast<uintptr_t>(x) ^ reinterpret_cast<uintptr_t>(g_out)) & 15) != 0) continue;  // consumers' element loop
      const uint4 *xbody = reinterpret_cast<const uint4 *>(x + head);
      for (int v0 = 0; v0 < nvec; v0 += STAGE_VECS) {
        const uint32_t bytes = static_cast<uint32_t>(min(STAGE_VECS, nvec - v0)) * 16u;
        while (it - retired >= LAG) retire_one();  // keep at most LAG chunks between load and store
        const int s = static_cast<int>(it % STAGES);
        // the stage's previous chunk (it - STAGES) was handed to the copy engine at least STAGES - LAG
        // stores ago: wait until the engine has finished READING it (later groups may stay pending)
        asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(STAGES - LAG) : "memory");
        st_dst[s] = reinterpret_cast<uint64_t>(gbody + v0);
        st_bytes[s] = bytes;
        bulk::mbar_expect_tx(full + s, bytes);
        bulk::bulk_g2s(ring + static_cast<size_t>(s) * STAGE_VECS, xbody + v0, bytes, full + s);
        ++it;
      }
    }
    while (retired < it) retire_one();
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // smem must outlive the engine's reads / the stores
    return;
  }

  // ------------------------------ consumer warps ------------------------------
  int64_t it = 0;
  for (int64_t r = blockIdx.x; r < n_work; r += gridDim.x) {
    const int4 *rv = reinterpret_cast<const int4 *>(rec) + r * kRecVecs;
    const int4 r0 = __ldg(rv);
    const int4 r1 = __ldg(rv + 1);
    const int y = r1.w;
    if (y == -2) continue;
    float H = 0.f, gH = 0.f;
    if constexpr (ENT) {
      const int4 r2 = __ldg(rv + 2);
      H = __int_as_float(r2.x);
      gH = __int_as_float(r2.y);
    }
    const bool ent = ENT && gH != 0.f;  // rows without an entropy gradient run the plain code
    const int64_t x_off = (static_cast<int64_t>(static_cast<uint32_t>(r0.y)) << 32) | static_cast<uint32_t>(r0.x);
    const int64_t g_row = (static_cast<int64_t>(static_cast<uint32_t>(r0.w)) << 32) | static_cast<uint32_t>(r0.z);
    const float m = __int_as_float(r1.x), logsum = __int_as_float(r1.y), g = __int_as_float(r1.z);
    T *g_out = grad + g_row * grad_row_stride;
    const T *x = logits + x_off;
    const float lse = m + logsum;
    const float c_f32 = -lse * kLog2e;
    const float neg_g = FAITHFUL ? -g : -g * ex2_approx(fmaf(-lse, kLog2e, -c_f32));
    const GradConsts gk = make_grad_consts(m, logsum, c_f32, neg_g, zero);
    // -g_H, with the F32 mode's offset residual folded in as for -g
    const float ngh = !ENT ? 0.f : FAITHFUL ? -gH : -gH * ex2_approx(fmaf(-lse, kLog2e, -c_f32));
    const EntConsts ek{f2_splat(H), f2_splat(ngh)};
    // element c of the row; ENT = false is grad_of itself
#define AA_K1B_ELEM(c)                                                                                        \
  (ENT ? grad_of_ent<T, FAITHFUL>(Traits<T>::to_float(x[c]), m, logsum, c_f32, neg_g, g, (c) == y, ent, ngh, H) \
       : grad_of<T, FAITHFUL>(Traits<T>::to_float(x[c]), m, logsum, c_f32, neg_g, g, (c) == y))
    if (((reinterpret_cast<uintptr_t>(x) ^ reinterpret_cast<uintptr_t>(g_out)) & 15) != 0) {
      for (int e = tid; e < V; e += CONSUMERS) g_out[e] = Traits<T>::from_float(AA_K1B_ELEM(e));
      continue;
    }
    const int mis = static_cast<int>((reinterpret_cast<uintptr_t>(g_out) & 15) / sizeof(T));
    const int head = mis ? min(E - mis, V) : 0;
    const int nvec = (V - head) / E;
    const int tail0 = head + nvec * E;
    if (tid < head) g_out[tid] = Traits<T>::from_float(AA_K1B_ELEM(tid));
    if (tid < V - tail0) g_out[tail0 + tid] = Traits<T>::from_float(AA_K1B_ELEM(tail0 + tid));
#undef AA_K1B_ELEM
    const int yv = (y >= head && y < tail0) ? (y - head) / E : -1;  // body vector holding the label column
    for (int v0 = 0; v0 < nvec; v0 += STAGE_VECS) {
      const int n = min(STAGE_VECS, nvec - v0);
      const int s = static_cast<int>(it % STAGES);
      bulk::mbar_wait(full + s, static_cast<uint32_t>((it / STAGES) & 1));
      uint4 *buf = ring + static_cast<size_t>(s) * STAGE_VECS;
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const int k = tid + u * CONSUMERS;
        if (k < n) {
          const uint4 in = buf[k];
          uint4 o = ent ? vec_grad_ent<T, FAITHFUL, false>(in, gk, ek) : vec_grad<T, FAITHFUL>(in, gk);
          if (v0 + k == yv)
            patch_label<T, FAITHFUL, ENT>(o, in, (y - head) - (v0 + k) * E, m, logsum, c_f32, neg_g, g, ent, ngh, H);
          buf[k] = o;
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the copy engine
      __syncwarp();
      if ((tid & 31) == 0) bulk::mbar_arrive(done + s);
      ++it;
    }
  }
}

// ---- host side ----------------------------------------------------------------------------
// Tuning knobs of the DIAGNOSTIC entry points aa_logprob_set_tuning{,_bwd}: process-wide by design (sweeps set them once,
// before a run; the trainers never touch them).  Atomics make a setter racing with launches on another thread well
// defined: such a launch may see the old or the new kernel, both valid -- results never depend on the knobs.
static std::atomic<int> g_variant{0};        // forward: 0 / 3 by row length, 1 ring, 2 LDG
static std::atomic<int> g_ctas_per_sm{0};
static std::atomic<int> g_bwd_variant{0};    // backward: -1 / 0 / 1 TMA-staged, 3 LDG row kernel
static std::atomic<int> g_bwd_ctas_per_sm{0};
static inline int fwd_variant() { return g_variant.load(std::memory_order_relaxed); }
static inline int fwd_ctas() { return g_ctas_per_sm.load(std::memory_order_relaxed); }
static inline int bwd_variant() { return g_bwd_variant.load(std::memory_order_relaxed); }
static inline int bwd_ctas() { return g_bwd_ctas_per_sm.load(std::memory_order_relaxed); }

// Persistent forward grids are sized to what is resident at once: a second wave of a grid-strided kernel streams
// its rows with fewer CTAs per SM.  The occupancy is asked once per kernel instance (`resident` is the caller's
// cache; the library runs on one device model).  The tuning's ctas_per_sm can only lower the count.
template <typename K>
static int fwd_grid(K kern, int threads, size_t smem, std::atomic<int> &resident, int64_t n_rows, unsigned &grid) {
  int per_sm = resident.load(std::memory_order_relaxed);
  if (per_sm == 0) {  // a race computes the same value twice, harmlessly
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem);
    if (e != cudaSuccess || per_sm < 1) {
      set_error("aa_logprob_fwd: no resident CTA of %d threads with %zu B of shared memory: %s", threads, smem,
                cudaGetErrorString(e));
      return e != cudaSuccess ? static_cast<int>(e) : AA_ERR_UNSUPPORTED;
    }
    resident.store(per_sm, std::memory_order_relaxed);
  }
  if (fwd_ctas() > 0 && fwd_ctas() < per_sm) per_sm = fwd_ctas();
  const int64_t g = static_cast<int64_t>(sm_count()) * per_sm;
  grid = static_cast<unsigned>(g < n_rows ? g : n_rows);
  return 0;
}

template <typename T, bool ENT>
static int launch_fwd_ldg(const FwdParams &p, cudaStream_t st) {
  constexpr int THREADS = 512, UNROLL = 4;
  auto kern = logprob_fwd_kernel<T, THREADS, UNROLL, ENT>;
  static std::atomic<int> resident{0};
  unsigned grid = 0;
  int rc = fwd_grid(kern, THREADS, 0, resident, p.n_rows, grid);
  if (rc) return rc;
  kern<<<grid, THREADS, 0, st>>>(p);
  return check_launch("aa_logprob_fwd(ldg)");
}

template <typename T, bool ENT>
static int launch_fwd_ring(const FwdParams &p, cudaStream_t st) {
  constexpr int CONSUMERS = 256, STAGES = 4, UNROLL = 4;  // 4 stages x 16 KB; 3 CTAs per SM are resident
  constexpr size_t smem = fwd_ring_smem<CONSUMERS, STAGES, UNROLL>();
  auto kern = logprob_fwd_ring_kernel<T, CONSUMERS, STAGES, UNROLL, ENT>;
  static std::atomic<int> resident{0};
  unsigned grid = 0;
  int rc = fwd_grid(kern, CONSUMERS + 32, smem, resident, p.n_rows, grid);
  if (rc) return rc;
  kern<<<grid, CONSUMERS + 32, smem, st>>>(p);
  return check_launch("aa_logprob_fwd");
}

// Which forward streams a row is decided by the row's length.  Measured on an H100 SXM at 400 W (DESIGN.md section
// 3.1): rows of 256 KB and more (V = 128257 / 156032 in bf16) move faster through the LDG kernel at 4 CTAs x 512
// threads per SM (C2: 5.7 ms against 5.9-6.1 ms for the ring), 64 KB rows (V = 32064) through the ring (C3: 0.55 ms
// against 0.62 ms).  Tuning variant 1 forces the ring, variant 2 the LDG kernel.
constexpr int64_t kFwdLdgMinRowBytes = 128 * 1024;

template <typename T, bool ENT = false>
static int launch_fwd(const FwdParams &p, cudaStream_t st) {
  const int variant = fwd_variant();
  if (variant == 2 || (variant != 1 && static_cast<int64_t>(p.V) * sizeof(T) >= kFwdLdgMinRowBytes))
    return launch_fwd_ldg<T, ENT>(p, st);
  return launch_fwd_ring<T, ENT>(p, st);
}

template <typename T, int THREADS, int UNROLL, bool FAITHFUL>
static int launch_bwd_shape(const BwdParams &p, int per_sm, cudaStream_t st) {
  const int64_t n_work = bwd_work_rows(p);
  int64_t grid = static_cast<int64_t>(sm_count()) * per_sm;
  if (grid > n_work) grid = n_work;
  logprob_bwd_kernel<T, THREADS, UNROLL, FAITHFUL><<<static_cast<unsigned>(grid), THREADS, 0, st>>>(p);
  return check_launch("aa_logprob_bwd");
}

// TMA-staged backward: 256 consumers, 4 stages x 8 KB, lag 3, 3 CTAs/SM.
template <typename T, bool ENT = false>
static int launch_bwd_tma(const BwdParams &p, int mode, RowRec *rec, cudaStream_t st) {
  constexpr int CONSUMERS = 256, STAGES = 4, UNROLL = 2, LAG = 3;
  const int64_t n_work = bwd_work_rows(p);
  bwd_row_prep_kernel<ENT><<<static_cast<unsigned>((n_work + 255) / 256), 256, 0, st>>>(p, rec);
  int rc = check_launch("aa_logprob_bwd(prep)");
  if (rc) return rc;
  constexpr size_t smem = static_cast<size_t>(STAGES + 1) * CONSUMERS * UNROLL * 16 + STAGES * (8 + 8 + 8 + 4) + 16;
  const bool faithful = (mode == AA_MODE_FAITHFUL) && sizeof(T) == 2;
  auto kf = logprob_bwd_tma_kernel<T, CONSUMERS, STAGES, UNROLL, LAG, true, ENT>;
  auto kn = logprob_bwd_tma_kernel<T, CONSUMERS, STAGES, UNROLL, LAG, false, ENT>;
  static std::atomic<bool> configured{false};  // the attribute is idempotent: a race sets it twice, harmlessly
  if (!configured.load(std::memory_order_relaxed)) {
    cudaError_t e = cudaFuncSetAttribute(kf, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(kn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) {
      set_error("aa_logprob_bwd(tma): cannot reserve %zu B of shared memory: %s", smem, cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    configured.store(true, std::memory_order_relaxed);
  }
  const int per_sm = bwd_ctas() > 0 ? bwd_ctas() : 3;
  int64_t grid = static_cast<int64_t>(sm_count()) * per_sm;
  if (grid > n_work) grid = n_work;
  const T *lg = reinterpret_cast<const T *>(p.logits);
  T *gr = reinterpret_cast<T *>(p.grad_logits);
  if (faithful)
    kf<<<static_cast<unsigned>(grid), CONSUMERS + 32, smem, st>>>(lg, gr, p.grad_row_stride, p.V, rec, n_work, p.zero);
  else
    kn<<<static_cast<unsigned>(grid), CONSUMERS + 32, smem, st>>>(lg, gr, p.grad_row_stride, p.V, rec, n_work, p.zero);
  return check_launch("aa_logprob_bwd(tma)");
}

// One-CTA-per-row LDG/STG backward.  The read+write stream is sensitive to how much is in flight per SM and the
// optimum depends on the compute per byte: 16-bit FAITHFUL (Veltkamp rounding, ~7 instr/elem) 512 thr x 4 vec x
// 3 CTAs/SM, 16-bit F32 mode (~3.5 instr/elem) 512 x 2 x 3, fp32 logits 256 x 4 x 4.
template <typename T>
static int launch_bwd(const BwdParams &p, int mode, cudaStream_t st) {
  const int c = bwd_ctas();
  if constexpr (sizeof(T) == 2) {
    if (mode == AA_MODE_FAITHFUL) return launch_bwd_shape<T, 512, 4, true>(p, c > 0 ? c : 3, st);
    return launch_bwd_shape<T, 512, 2, false>(p, c > 0 ? c : 3, st);
  }
  return launch_bwd_shape<T, 256, 4, false>(p, c > 0 ? c : 4, st);
}

}  // namespace aa

using namespace aa;

extern "C" int aa_logprob_set_tuning(int variant, int ctas_per_sm) {
  AA_REQUIRE(variant >= 0 && variant <= 3, AA_ERR_ARG,
             "aa_logprob_set_tuning: variant = 0 / 3 (by row length), 1 (ring) or 2 (LDG)");
  g_variant = variant;
  g_ctas_per_sm = ctas_per_sm;
  return AA_OK;
}

extern "C" int aa_logprob_set_tuning_bwd(int variant, int ctas_per_sm) {
  AA_REQUIRE(variant == -1 || variant == 0 || variant == 1 || variant == 3, AA_ERR_ARG,
             "aa_logprob_set_tuning_bwd: variant = -1 / 0 / 1 (TMA-staged) or 3 (LDG row kernel)");
  g_bwd_variant = variant;
  g_bwd_ctas_per_sm = ctas_per_sm;
  return AA_OK;
}

static int logprob_fwd(const char *who, const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                       const int64_t *labels, int64_t ignore_index, int32_t use_ignore, int32_t n_segments,
                       int64_t n_rows, const int64_t *seg_logit_off, const int64_t *seg_label_off,
                       const int64_t *seg_out_off, const int64_t *seg_cum, void *out, int out_dtype, float *stat_max,
                       float *stat_logsum, int32_t *status, float *entropy, int64_t n_entropy, void *stream) {
  AA_REQUIRE(V > 0 && n_segments >= 0 && n_rows >= 0, AA_ERR_ARG, "%s: bad sizes", who);
  if (n_rows == 0 || n_segments == 0) return AA_OK;
  AA_REQUIRE(logits && labels && out && seg_logit_off && seg_label_off && seg_out_off && seg_cum,
             AA_ERR_ARG, "%s: null pointer", who);
  AA_REQUIRE((stat_max == nullptr) == (stat_logsum == nullptr), AA_ERR_ARG,
             "%s: stat_max and stat_logsum go together", who);
  AA_REQUIRE(out_dtype == AA_BF16 || out_dtype == AA_F16 || out_dtype == AA_F32, AA_ERR_DTYPE,
             "%s: bad out_dtype %d", who, out_dtype);
  const int esz = dtype_size(logits_dtype);
  AA_REQUIRE(reinterpret_cast<uintptr_t>(logits) % esz == 0, AA_ERR_ALIGN,
             "%s: logits not element-aligned", who);
  FwdParams p{logits, row_stride, V, labels, ignore_index, use_ignore,
              RowMap{seg_logit_off, seg_label_off, seg_out_off, seg_cum, n_segments},
              n_rows, out, out_dtype, stat_max, stat_logsum, status, kLog2e, entropy, n_entropy};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (entropy) {
    switch (logits_dtype) {
      case AA_BF16: return launch_fwd<__nv_bfloat16, true>(p, st);
      case AA_F16: return launch_fwd<__half, true>(p, st);
      case AA_F32: return launch_fwd<float, true>(p, st);
    }
  } else {
    switch (logits_dtype) {
      case AA_BF16: return launch_fwd<__nv_bfloat16>(p, st);
      case AA_F16: return launch_fwd<__half>(p, st);
      case AA_F32: return launch_fwd<float>(p, st);
    }
  }
  set_error("%s: unsupported logits dtype %d", who, logits_dtype);
  return AA_ERR_DTYPE;
}

extern "C" int aa_logprob_fwd(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                              const int64_t *labels, int64_t ignore_index, int32_t use_ignore,
                              int32_t n_segments, int64_t n_rows,
                              const int64_t *seg_logit_off, const int64_t *seg_label_off,
                              const int64_t *seg_out_off, const int64_t *seg_cum, void *out,
                              int out_dtype, float *stat_max, float *stat_logsum, int32_t *status,
                              void *stream) {
  return logprob_fwd("aa_logprob_fwd", logits, logits_dtype, row_stride, V, labels, ignore_index, use_ignore,
                     n_segments, n_rows, seg_logit_off, seg_label_off, seg_out_off, seg_cum, out, out_dtype, stat_max,
                     stat_logsum, status, nullptr, 0, stream);
}

extern "C" int aa_logprob_fwd_entropy(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                      const int64_t *labels, int64_t ignore_index, int32_t use_ignore,
                                      int32_t n_segments, int64_t n_rows,
                                      const int64_t *seg_logit_off, const int64_t *seg_label_off,
                                      const int64_t *seg_out_off, const int64_t *seg_cum, void *out,
                                      int out_dtype, float *stat_max, float *stat_logsum, int32_t *status,
                                      float *entropy, int64_t n_entropy, void *stream) {
  AA_REQUIRE(entropy && n_entropy >= 0, AA_ERR_ARG, "aa_logprob_fwd_entropy: null entropy");
  return logprob_fwd("aa_logprob_fwd_entropy", logits, logits_dtype, row_stride, V, labels, ignore_index, use_ignore,
                     n_segments, n_rows, seg_logit_off, seg_label_off, seg_out_off, seg_cum, out, out_dtype, stat_max,
                     stat_logsum, status, entropy, n_entropy, stream);
}

extern "C" int aa_zero_rows(void *tile, int dtype, int64_t row_stride, int32_t V, int64_t n_tile_rows,
                            const int64_t *spans_host, int32_t n_spans, void *stream) {
  AA_REQUIRE(V > 0 && row_stride >= V && n_spans >= 0 && n_tile_rows >= 0, AA_ERR_ARG, "aa_zero_rows: bad sizes");
  if (n_spans == 0) return AA_OK;
  AA_REQUIRE(tile && spans_host, AA_ERR_ARG, "aa_zero_rows: null pointer");
  AA_REQUIRE(dtype == AA_BF16 || dtype == AA_F16 || dtype == AA_F32, AA_ERR_DTYPE, "aa_zero_rows: bad dtype");
  const size_t esz = (dtype == AA_F32) ? 4 : 2;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uintptr_t lo = reinterpret_cast<uintptr_t>(tile);
  const uintptr_t hi = lo + static_cast<size_t>(n_tile_rows) * V * esz;  // contiguous tiles only
  constexpr uintptr_t kAlign = 256;
  for (int32_t i = 0; i < n_spans; ++i) {
    const int64_t first = spans_host[2 * i], n = spans_host[2 * i + 1];
    AA_REQUIRE(first >= 0 && n >= 0 && first + n <= n_tile_rows, AA_ERR_ARG, "aa_zero_rows: bad span %d", i);
    if (n == 0) continue;
    cudaError_t e;
    if (row_stride == V) {
      // Rows of an odd vocabulary (V = 128257) start 2-byte aligned, and a memset whose ends are not aligned runs
      // at a fraction of the copy engine's rate.  The rows next to a span are rewritten in full by the kernel that
      // follows in stream order, so the span is widened to 256-byte boundaries (inside the tile).
      uintptr_t a = (lo + static_cast<size_t>(first) * V * esz) & ~(kAlign - 1);
      uintptr_t b = (lo + static_cast<size_t>(first + n) * V * esz + kAlign - 1) & ~(kAlign - 1);
      if (a < lo) a = lo;
      if (b > hi) b = hi;
      e = cudaMemsetAsync(reinterpret_cast<void *>(a), 0, b - a, st);
    } else {
      char *dst = static_cast<char *>(tile) + static_cast<size_t>(first) * row_stride * esz;
      e = cudaMemset2DAsync(dst, static_cast<size_t>(row_stride) * esz, 0, static_cast<size_t>(V) * esz,
                            static_cast<size_t>(n), st);
    }
    if (e != cudaSuccess) {
      set_error("aa_zero_rows: %s", cudaGetErrorString(e));
      return static_cast<int>(e);
    }
  }
  return AA_OK;
}

// aa_logprob_bwd{,_entropy}: entropy == nullptr runs the plain kernels
static int logprob_bwd(const char *who, const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                       const int64_t *labels, int64_t ignore_index, int32_t use_ignore, int32_t n_segments,
                       int64_t n_rows, const int64_t *seg_logit_off, const int64_t *seg_label_off,
                       const int64_t *seg_out_off, const int64_t *seg_cum, const int64_t *seg_tile_row,
                       const float *stat_max, const float *stat_logsum, const void *grad_rows, int grad_rows_dtype,
                       const float *grad_seg, const void *grad_scale, int grad_scale_dtype, void *grad_logits,
                       int64_t grad_row_stride, int64_t n_tile_rows, const int64_t *extra_zero_rows,
                       int64_t n_extra_zero_rows, const float *entropy, const void *grad_entropy,
                       int grad_entropy_dtype, void *row_scratch, int mode, void *stream) {
  AA_REQUIRE(V > 0 && n_segments >= 0 && n_rows >= 0 && n_tile_rows >= 0 && n_extra_zero_rows >= 0, AA_ERR_ARG,
             "%s: bad sizes", who);
  AA_REQUIRE(n_extra_zero_rows == 0 || (n_tile_rows == 0 && extra_zero_rows), AA_ERR_ARG,
             "%s: extra_zero_rows needs n_tile_rows == 0 and a device row list", who);
  if (n_segments == 0) n_rows = 0;
  if (n_tile_rows == 0 && n_rows == 0 && n_extra_zero_rows == 0) return AA_OK;
  AA_REQUIRE(grad_logits, AA_ERR_ARG, "%s: null grad_logits", who);
  if (n_segments > 0)
    AA_REQUIRE(logits && labels && seg_logit_off && seg_label_off && seg_out_off && seg_cum &&
                   seg_tile_row && stat_max && stat_logsum,
               AA_ERR_ARG, "%s: null pointer", who);
  AA_REQUIRE(mode == AA_MODE_FAITHFUL || mode == AA_MODE_F32, AA_ERR_ARG, "%s: bad mode", who);
  AA_REQUIRE(!grad_scale || grad_scale_dtype == AA_BF16 || grad_scale_dtype == AA_F16 || grad_scale_dtype == AA_F32,
             AA_ERR_DTYPE, "%s: bad grad_scale dtype", who);
  BwdParams p{logits, row_stride, V, labels, ignore_index, use_ignore,
              RowMap{seg_logit_off, seg_label_off, seg_out_off, seg_cum, n_segments},
              n_rows, seg_tile_row, stat_max, stat_logsum, grad_rows, grad_rows_dtype, grad_seg,
              grad_scale, grad_scale_dtype, grad_logits, grad_row_stride, n_tile_rows, 0.0f, extra_zero_rows, n_extra_zero_rows,
              entropy, grad_entropy, grad_entropy_dtype};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (entropy) {  // the TMA-staged kernel only (the caller checked row_scratch)
    AA_REQUIRE((reinterpret_cast<uintptr_t>(row_scratch) & 15) == 0, AA_ERR_ALIGN,
               "%s: row_scratch must be 16-byte aligned", who);
    RowRec *rec = static_cast<RowRec *>(row_scratch);
    switch (logits_dtype) {
      case AA_BF16: return launch_bwd_tma<__nv_bfloat16, true>(p, mode, rec, st);
      case AA_F16: return launch_bwd_tma<__half, true>(p, mode, rec, st);
      case AA_F32: return launch_bwd_tma<float, true>(p, mode, rec, st);
    }
    set_error("%s: unsupported logits dtype %d", who, logits_dtype);
    return AA_ERR_DTYPE;
  }
  if (row_scratch && bwd_variant() != 3) {  // TMA-staged backward (the default); tuning variant 3 takes the LDG kernel
    AA_REQUIRE((reinterpret_cast<uintptr_t>(row_scratch) & 15) == 0, AA_ERR_ALIGN,
               "aa_logprob_bwd: row_scratch must be 16-byte aligned");
    RowRec *rec = static_cast<RowRec *>(row_scratch);
    switch (logits_dtype) {
      case AA_BF16: return launch_bwd_tma<__nv_bfloat16>(p, mode, rec, st);
      case AA_F16: return launch_bwd_tma<__half>(p, mode, rec, st);
      case AA_F32: return launch_bwd_tma<float>(p, mode, rec, st);
    }
  }
  switch (logits_dtype) {
    case AA_BF16: return launch_bwd<__nv_bfloat16>(p, mode, st);
    case AA_F16: return launch_bwd<__half>(p, mode, st);
    case AA_F32: return launch_bwd<float>(p, mode, st);
  }
  set_error("%s: unsupported logits dtype %d", who, logits_dtype);
  return AA_ERR_DTYPE;
}

extern "C" int aa_logprob_bwd(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                              const int64_t *labels, int64_t ignore_index, int32_t use_ignore,
                              int32_t n_segments, int64_t n_rows,
                              const int64_t *seg_logit_off, const int64_t *seg_label_off,
                              const int64_t *seg_out_off, const int64_t *seg_cum,
                              const int64_t *seg_tile_row, const float *stat_max,
                              const float *stat_logsum, const void *grad_rows, int grad_rows_dtype,
                              const float *grad_seg, const void *grad_scale, int grad_scale_dtype, void *grad_logits,
                              int64_t grad_row_stride, int64_t n_tile_rows, const int64_t *extra_zero_rows,
                              int64_t n_extra_zero_rows, void *row_scratch, int mode, void *stream) {
  return logprob_bwd("aa_logprob_bwd", logits, logits_dtype, row_stride, V, labels, ignore_index, use_ignore, n_segments,
                     n_rows, seg_logit_off, seg_label_off, seg_out_off, seg_cum, seg_tile_row, stat_max, stat_logsum,
                     grad_rows, grad_rows_dtype, grad_seg, grad_scale, grad_scale_dtype, grad_logits, grad_row_stride,
                     n_tile_rows, extra_zero_rows, n_extra_zero_rows, nullptr, nullptr, AA_F32, row_scratch, mode,
                     stream);
}

extern "C" int aa_logprob_bwd_entropy(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                      const int64_t *labels, int64_t ignore_index, int32_t use_ignore,
                                      int32_t n_segments, int64_t n_rows,
                                      const int64_t *seg_logit_off, const int64_t *seg_label_off,
                                      const int64_t *seg_out_off, const int64_t *seg_cum,
                                      const int64_t *seg_tile_row, const float *stat_max,
                                      const float *stat_logsum, const void *grad_rows, int grad_rows_dtype,
                                      const float *grad_seg, const void *grad_scale, int grad_scale_dtype,
                                      const float *entropy, const void *grad_entropy, int grad_entropy_dtype,
                                      void *grad_logits, int64_t grad_row_stride, int64_t n_tile_rows,
                                      const int64_t *extra_zero_rows, int64_t n_extra_zero_rows, void *row_scratch,
                                      int mode, void *stream) {
  AA_REQUIRE(entropy && grad_entropy && row_scratch, AA_ERR_ARG,
             "aa_logprob_bwd_entropy: entropy, grad_entropy and row_scratch (48 bytes per work row) are required");
  AA_REQUIRE(grad_entropy_dtype == AA_BF16 || grad_entropy_dtype == AA_F16 || grad_entropy_dtype == AA_F32,
             AA_ERR_DTYPE, "aa_logprob_bwd_entropy: bad grad_entropy dtype");
  return logprob_bwd("aa_logprob_bwd_entropy", logits, logits_dtype, row_stride, V, labels, ignore_index, use_ignore,
                     n_segments, n_rows, seg_logit_off, seg_label_off, seg_out_off, seg_cum, seg_tile_row, stat_max,
                     stat_logsum, grad_rows, grad_rows_dtype, grad_seg, grad_scale, grad_scale_dtype, grad_logits,
                     grad_row_stride, n_tile_rows, extra_zero_rows, n_extra_zero_rows, entropy, grad_entropy,
                     grad_entropy_dtype, row_scratch, mode, stream);
}
