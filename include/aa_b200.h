/*
 * aa_b200.h -- C ABI of libaa_b200.so: the H100 (sm_90a) implementation of
 * align-anything's RLHF loss hot path.
 *
 * The reference (PKU-Alignment/align-anything) has NO FFI layer for this path:
 * the boundary is plain Python (module-level helpers in align_anything/utils/tools.py
 * and methods on the trainer classes).  Each entry point below names the reference
 * function(s) whose arithmetic it replaces (file:line relative to the reference's
 * align_anything/ directory); the Python mirror in align_anything_b200/ keeps the
 * reference's names and signatures and calls these through ctypes (INTEGRATION.md).
 * 82 entry points, ABI version 3.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - the caller owns every buffer (inputs, outputs, scratch); the library allocates
 *     nothing and keeps no state besides a thread-local error string;
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*); no entry
 *     point synchronises the host;
 *   - return value: 0 on success, AA_ERR_* (<0) for argument errors, or a positive
 *     cudaError_t from the launch.  aa_last_error() gives the text;
 *   - offsets / strides are in ELEMENTS of the tensor they index;
 *   - `mode`: AA_MODE_FAITHFUL reproduces the reference's rounding points when the
 *     tensors are bf16/f16 (fp32 arithmetic, round-to-nearest-even to the tensor dtype
 *     where the reference's eager ops round); AA_MODE_F32 keeps fp32 throughout.
 */
#ifndef AA_B200_H_
#define AA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AA_B200_ABI_VERSION 3

enum { AA_BF16 = 0, AA_F16 = 1, AA_F32 = 2 };
enum { AA_MODE_FAITHFUL = 0, AA_MODE_F32 = 1 };
enum { AA_MASK_U8 = 0, AA_MASK_I64 = 1 };

enum {
  AA_OK = 0,
  AA_ERR_DTYPE = -1,
  AA_ERR_ARG = -2,
  AA_ERR_ALIGN = -3,
  AA_ERR_UNSUPPORTED = -4
};

/* bits OR-ed into the device status word by kernels (never cleared by the library) */
enum {
  AA_STATUS_LABEL_OOB = 1,      /* a label outside [0, V): torch.gather would raise           */
  AA_STATUS_SHORT_SEQUENCE = 2, /* fewer non-pad tokens than response_len (dpo.py:135-137)   */
  AA_STATUS_EMPTY_MASK = 4,     /* a mask row with no True: m.nonzero()[-1] would raise       */
  AA_STATUS_DIVERGE_RANGE = 8,  /* simpo.py:72-73 `assert 0 <= diverge_index <= end_index` fails */
  AA_STATUS_WHITEN_COUNT = 16   /* fewer than 2 masked advantages to whiten (verl's masked_var raises) */
};

/* Descriptor of the one-shot NVLink all-reduce fused into the metric-producing kernels (multi-GPU only).
 * peer_bufs: DEVICE array [world] of peer-mapped pointers to each rank's symmetric buffer of
 * 2 * world * 16 floats + world uint32 flags, zero-initialised once (torch.distributed._symmetric_memory
 * gives such pointers).  epoch: 1, 2, 3, ... incremented by the caller on every use, identically on every
 * rank.  max_lanes: bit t set -> lane t is MAX-reduced, otherwise averaged (utils/multi_process.py:74-89). */
typedef struct aa_coll {
  void *const *peer_bufs;
  int32_t rank;
  int32_t world;
  uint32_t epoch;
  uint32_t max_lanes;
} aa_coll;

int aa_abi_version(void);
const char *aa_last_error(void);
/* Number of SMs / max dynamic smem of the current device (for host-side grid sizing). */
int aa_device_info(int *sm_count, int *max_smem_optin);
/* Tuning / diagnostic knobs (process-wide).  Each kernel has one launch shape; the variant only picks the kernel.
 *   K1 forward (aa_logprob_set_tuning): 0 / 3 = chosen by row length (default), 1 = cp.async.bulk ring through
 *            shared memory, 2 = vectorised LDG; the grid is the resident CTA count.
 *   K1b backward (aa_logprob_set_tuning_bwd): -1 / 0 / 1 = TMA-staged (cp.async.bulk loads AND stores through a
 *            shared-memory ring, 4 stages x 8 KB, lag 3, 3 CTAs/SM; the default whenever row_scratch is given),
 *            3 = one-CTA-per-row LDG/STG kernel (also used when row_scratch == NULL).
 * Any other variant is AA_ERR_ARG.  ctas_per_sm <= 0 keeps the default persistent-grid size; the forward's can only
 * lower it. */
int aa_logprob_set_tuning(int variant, int ctas_per_sm);
/* Same, for K1b only; the two settings are independent. */
int aa_logprob_set_tuning_bwd(int variant, int ctas_per_sm);

/* ---------------------------------------------------------------------------------------
 * K1  per-token log-prob: row log-softmax over V fused with the label gather.
 * Replaces utils/tools.py:402-413 gather_log_probabilities and the per-sample slicing loop
 * around it (trainers/text_to_text/dpo.py:133-142, text_image_to_text/ppo.py:229-239).
 *
 * A "segment" is one run of consecutive logits rows scored against consecutive labels
 * (one sample's response tail, or one whole sample).  Segment s covers flat rows
 * [seg_cum[s], seg_cum[s+1]); its j-th row reads logits[seg_logit_off[s] + j*row_stride + 0..V),
 * label labels[seg_label_off[s] + j], and writes out[seg_out_off[s] + j].
 *
 *   out         : out_dtype (the logits dtype in FAITHFUL mode -> same rounding as
 *                 F.log_softmax's output; AA_F32 otherwise)
 *   stat_max, stat_logsum : optional fp32 [n_rows] (flat row order) saved for K1b.
 *   status      : optional device int32 word, see AA_STATUS_*.
 *   use_ignore  : != 0 -> rows whose label == ignore_index are skipped (out = 0, no traffic; K1b
 *                 zero-fills them): the cross-entropy `ignore_index` of the SFT / PTX loss.
 * Algorithmic HBM traffic: V * sizeof(logit) bytes per row, read once.
 * ------------------------------------------------------------------------------------- */
int aa_logprob_fwd(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                   const int64_t *labels, int64_t ignore_index, int32_t use_ignore,
                   int32_t n_segments, int64_t n_rows,
                   const int64_t *seg_logit_off, const int64_t *seg_label_off,
                   const int64_t *seg_out_off, const int64_t *seg_cum,
                   void *out, int out_dtype, float *stat_max, float *stat_logsum,
                   int32_t *status, void *stream);

/* K1 with the policy entropy of every scored row: aa_logprob_fwd's arguments (same outputs, bit for bit) plus
 *   entropy   : fp32, H = -sum_j p_j log p_j of the row's fp32-upcast logits, written at the row's OUT position
 *               (never rounded to out_dtype).  Only rows whose out position is < n_entropy are written: with a two-copy
 *               plan (aa_tail_plan_build, copies = 2) n_entropy = copy_out_delta keeps the entropy of the first copy
 *               and the buffer needs no room for the second.  Ignored rows (use_ignore) get 0; rows the plan does not
 *               score are not written (the caller zero-initialises); an all -inf row gets NaN; a -inf logit adds 0.
 * One more FMA (and a clamp) per logit on top of the online (max, sum-exp): t = sum_j e^{x_j - m} (x_j - m), H = log s - t / s. */
int aa_logprob_fwd_entropy(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                           const int64_t *labels, int64_t ignore_index, int32_t use_ignore,
                           int32_t n_segments, int64_t n_rows,
                           const int64_t *seg_logit_off, const int64_t *seg_label_off,
                           const int64_t *seg_out_off, const int64_t *seg_cum,
                           void *out, int out_dtype, float *stat_max, float *stat_logsum,
                           int32_t *status, float *entropy, int64_t n_entropy, void *stream);

/* ---------------------------------------------------------------------------------------
 * K1b  d(log-prob)/d(logits): autograd of the two ops above (ATen _log_softmax_backward_data
 * + gather backward) in ONE pass: grad[j] = g * ([j == label] - softmax_j), written in the
 * logits dtype.  g for flat row r of segment s is
 *     (grad_rows ? grad_rows[seg_out_off[s] + j] : 1) * (grad_seg ? grad_seg[s] : 1)
 *                                                   * (grad_scale ? *grad_scale : 1)
 * (grad_scale: one device scalar of dtype grad_scale_dtype -- the upstream d loss of a fused loss node, read as it is).
 * The gradient tile is `n_tile_rows` rows of `grad_row_stride` elements; segment s owns tile
 * rows [seg_tile_row[s], seg_tile_row[s] + n_s) (ascending, non-overlapping); every other
 * tile row is ZERO-FILLED by the same kernel (the reference's autograd materialises those
 * zeros through the slice / pad backward).  n_tile_rows == 0: only scored rows are written,
 * at grad_logits + seg_tile_row[s]*grad_row_stride, followed by the `n_extra_zero_rows` tile rows
 * listed in `extra_zero_rows` (device, int64), which are zero-filled.  A caller that knows the row
 * layout on the host uses this form together with aa_zero_rows: long zero spans go to the copy
 * engine (cudaMemsetAsync, faster than stores issued by a kernel), isolated
 * zero rows are listed, and the kernel's static row stride sees equally expensive rows first.
 * FAITHFUL mode recomputes softmax_j as exp(round_dtype((x_j - max) - logsum)), which is what
 * the reference's backward sees (it re-reads the ROUNDED log-softmax output).
 * row_scratch: 16-byte aligned device scratch of 32 bytes per work row (n_tile_rows, or
 * n_rows + n_extra_zero_rows when n_tile_rows == 0).  With it the backward is TMA-staged: a tiny prep kernel resolves every row into a
 * 32-byte record, then a persistent kernel moves the tile with cp.async.bulk in both directions through
 * a shared-memory ring (6.48 TB/s sustained at V = 128257 vs 5.8 TB/s for the LDG/STG kernel).
 * row_scratch == NULL (or tuning variant 3) runs the one-CTA-per-row LDG/STG kernel, which computes the
 * same tile bit for bit.
 * Algorithmic HBM traffic: 2 * V * sizeof(logit) per scored row (+ V * sizeof per zero row).
 * ------------------------------------------------------------------------------------- */
int aa_logprob_bwd(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                   const int64_t *labels, int64_t ignore_index, int32_t use_ignore,
                   int32_t n_segments, int64_t n_rows,
                   const int64_t *seg_logit_off, const int64_t *seg_label_off,
                   const int64_t *seg_out_off, const int64_t *seg_cum,
                   const int64_t *seg_tile_row,
                   const float *stat_max, const float *stat_logsum,
                   const void *grad_rows, int grad_rows_dtype, const float *grad_seg,
                   const void *grad_scale, int grad_scale_dtype,
                   void *grad_logits, int64_t grad_row_stride, int64_t n_tile_rows,
                   const int64_t *extra_zero_rows, int64_t n_extra_zero_rows,
                   void *row_scratch, int mode, void *stream);

/* aa_logprob_bwd with the gradient of the rows' entropy added (entropy bonus): the tile element becomes
 *   g * (onehot_y - p_k)  -  g_H * p_k * (l_k + H),   l_k = x_k - max - logsum, p_k = e^{l_k}
 * with p_k and l_k as the log-prob term uses them (FAITHFUL: the rounded log-softmax), the correction in fp32 before the
 * tile's one rounding, and 0 for a -inf logit.  entropy: the fp32 H of aa_logprob_fwd_entropy; grad_entropy: g_H in
 * grad_entropy_dtype; both indexed like grad_rows.  grad_scale multiplies g_H too, grad_seg does not.  A row with
 * g_H == 0 is bit-identical to aa_logprob_bwd's.  row_scratch is required: 48 bytes per work row, 16-byte aligned.
 * This entry always runs the TMA-staged kernel: the LDG row kernel (aa_logprob_set_tuning_bwd variant 3) has no
 * entropy variant, and the tuning does not apply here. */
int aa_logprob_bwd_entropy(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                           const int64_t *labels, int64_t ignore_index, int32_t use_ignore,
                           int32_t n_segments, int64_t n_rows,
                           const int64_t *seg_logit_off, const int64_t *seg_label_off,
                           const int64_t *seg_out_off, const int64_t *seg_cum,
                           const int64_t *seg_tile_row,
                           const float *stat_max, const float *stat_logsum,
                           const void *grad_rows, int grad_rows_dtype, const float *grad_seg,
                           const void *grad_scale, int grad_scale_dtype,
                           const float *entropy, const void *grad_entropy, int grad_entropy_dtype,
                           void *grad_logits, int64_t grad_row_stride, int64_t n_tile_rows,
                           const int64_t *extra_zero_rows, int64_t n_extra_zero_rows,
                           void *row_scratch, int mode, void *stream);

/* Zero-fill row spans of an (n_tile_rows, V) tile with the copy engine.  spans_host: n_spans pairs
 * (first_row, n_rows) in HOST memory (read during the call); rows are row_stride elements apart.
 * Used for the prompt / padding rows of the gradient tile, BEFORE aa_logprob_bwd on the same stream:
 * for a contiguous tile (row_stride == V) each span is widened to 256-byte boundaries inside the tile
 * (an unaligned memset runs far below the copy engine's rate and rows of an odd V start 2-byte
 * aligned), i.e. up to 255 bytes of the neighbouring rows are cleared too -- aa_logprob_bwd rewrites
 * those rows in full afterwards.  Pitched tiles (row_stride > V) are cleared exactly. */
int aa_zero_rows(void *tile, int dtype, int64_t row_stride, int32_t V, int64_t n_tile_rows,
                 const int64_t *spans_host, int32_t n_spans, void *stream);

/* ---------------------------------------------------------------------------------------
 * Label extraction for DPO: labels of sample i = strip_pad(input_ids[i])[-R_i:]
 * (trainers/text_to_text/dpo.py:52-54, :135-137): the last R_i tokens that are != pad,
 * wherever the pads sit.  strip == 0 reproduces text_audio_to_text/dpo.py:100 (plain tail).
 * Writes labels_out[i*out_stride + k], k in [0, R_i) (bit-exact int64 copy).
 * ------------------------------------------------------------------------------------- */
int aa_strip_pad_tail(const int64_t *input_ids, int32_t n_samples, int32_t L, int64_t ids_row_stride,
                      int64_t pad_id, int strip, const int32_t *response_lens,
                      int64_t *labels_out, int64_t out_stride, int32_t *status, void *stream);

/* ---------------------------------------------------------------------------------------
 * K2  DPO pairwise loss + metrics.  Replaces trainers/text_to_text/dpo.py:166-203 (loss) and
 * :215-221 (local means); text_audio_to_text/dpo.py:134-139 when `input_ids` != NULL (pairs
 * whose chosen / rejected id rows are identical are dropped).
 *   policy_lp, ref_lp : (2*n_pairs, width), rows 0..n_pairs-1 chosen, rest rejected, zero padded.
 *   per_pair : fp32 [5][n_pairs] = loss_i, better_reward_i, worse_reward_i,
 *              g_i (= d mean-loss / d chosen-logp-sum_i ; rejected gets -g_i), valid_i (0/1).
 *   grad_seg : optional fp32 [2*n_pairs] = (+g_i ..., -g_i ...) ready for aa_logprob_bwd.
 *   stats    : fp32 [8] = loss, reward, better_sample_reward, worse_sample_reward,
 *              reward_accuracy, reward_margin (all means over valid pairs), n_valid, status.
 *   status   : optional device status word (AA_STATUS_* bits set by K1 / the label kernels earlier on the
 *              stream); its value is copied into stats[7] so that the caller's ONE host read of the metrics
 *              also tells it whether the reference would have raised (lane 7 is MAX-reduced across ranks).
 *   counter  : device uint32 scratch, zero before first use (the kernel re-zeroes it).
 *   coll / stats_global : optional (NULL on one GPU).  With them the last block of K2 also performs the
 *              step's packed all-reduce (trainers/text_to_text/dpo.py:222-227) over NVLink peer memory and
 *              writes the reduced vector to stats_global[8]; `stats` always holds the LOCAL values (the
 *              loss that is back-propagated is the local mean, as in the reference).
 * ------------------------------------------------------------------------------------- */
int aa_dpo_loss(const void *policy_lp, const void *ref_lp, int lp_dtype, int32_t n_pairs,
                int32_t width, int64_t lp_row_stride, float scale_coeff, int mode,
                const int64_t *input_ids, int32_t L, int64_t ids_row_stride,
                float *per_pair, float *grad_seg, float *stats, uint32_t *counter,
                const aa_coll *coll, float *stats_global, const int32_t *status, void *stream);

/* ---------------------------------------------------------------------------------------
 * K2 with the objective options of TRL's DPOConfig (DESIGN.md section 4.5): loss_type, label_smoothing
 * (cDPO / robust DPO), rpo_alpha (RPO's NLL term) and reference-free DPO.  With a = pc - rc, b = pr - rr (the
 * policy / reference log-prob sums of the chosen / rejected rows), h = a - b, z = scale_coeff * h:
 *   AA_DPO_SIGMOID    -(1-e) logsig(z) - e logsig(-z)            (e = label_smoothing; e = 0: aa_dpo_loss's loss)
 *   AA_DPO_ROBUST     (-(1-e) logsig(z) + e logsig(-z)) / (1 - 2e)
 *   AA_DPO_HINGE      relu(1 - z)
 *   AA_DPO_IPO        (h - 1/(2 beta))^2, each of the four sums divided by its row's counts[] entry first
 *   AA_DPO_SPPO_HARD  (a - 1/(2 beta))^2 + (b + 1/(2 beta))^2
 *   AA_DPO_NCA_PAIR   -logsig(beta a) - logsig(-beta a) / 2 - logsig(-beta b) / 2
 *   AA_DPO_APO_ZERO   (1 - sigmoid(beta a)) + sigmoid(beta b)
 *   AA_DPO_APO_DOWN   sigmoid(beta a) + (1 - sigmoid(beta h))
 * loss = mean over kept pairs; rpo_alpha > 0 adds rpo_alpha * NLL, NLL = -sum(pc) / sum(counts of those chosen rows)
 * over the kept pairs, and stats has a 9th lane = NLL.  ref_lp == NULL: reference-free (rc = rr = 0, nothing read).
 *   counts   : int32 [2*n_pairs] scored rows per sample (R_i - 1); needed by AA_DPO_IPO and rpo_alpha > 0.
 *   per_pair : as aa_dpo_loss, g_i = d loss / d chosen sum_i.
 *   grad_seg : required, fp32 [2*n_pairs] = (d loss / d chosen sum ..., d loss / d rejected sum ...) for
 *              aa_logprob_bwd; the rejected seeds are no longer -g_i.
 *   stats    : fp32 [8] as aa_dpo_loss (stats[0] = the loss with the NLL term), [9] when rpo_alpha > 0.
 * Metrics keep aa_dpo_loss's definitions (from the summed ratios) for every loss type.  No collective: the caller
 * all-reduces stats.  label_smoothing must lie in [0, 0.5) and be 0 unless the type is SIGMOID or ROBUST;
 * rpo_alpha >= 0; IPO and SPPO_HARD need scale_coeff > 0.
 * ------------------------------------------------------------------------------------- */
enum {
  AA_DPO_SIGMOID = 0,
  AA_DPO_ROBUST = 1,
  AA_DPO_HINGE = 2,
  AA_DPO_IPO = 3,
  AA_DPO_SPPO_HARD = 4,
  AA_DPO_NCA_PAIR = 5,
  AA_DPO_APO_ZERO = 6,
  AA_DPO_APO_DOWN = 7
};
int aa_dpo_loss_obj(const void *policy_lp, const void *ref_lp, int lp_dtype, int32_t n_pairs, int32_t width,
                    int64_t lp_row_stride, float scale_coeff, int mode, int loss_type, float label_smoothing,
                    float rpo_alpha, const int32_t *counts, const int64_t *input_ids, int32_t L,
                    int64_t ids_row_stride, float *per_pair, float *grad_seg, float *stats, uint32_t *counter,
                    const int32_t *status, void *stream);

/* ---------------------------------------------------------------------------------------
 * K2 with the further objectives of TRL's DPOConfig (DESIGN.md section 4.13): aa_dpo_loss_obj's arguments and
 * arithmetic, plus f-divergences (f_divergence_type) and the loss types below.  With a, b, h as above and
 * e = label_smoothing:
 *   f_divergence (replaces h; only for SIGMOID, ROBUST, HINGE and EXO_PAIR):
 *     AA_DPO_FDIV_REVERSE_KL  h = a - b                                       (aa_dpo_loss_obj's h)
 *     AA_DPO_FDIV_JS          h = (a - b) - (softplus(a) - softplus(b))
 *     AA_DPO_FDIV_ALPHA       h = (cap_exp(-f_alpha_coef b) - cap_exp(-f_alpha_coef a)) / f_alpha_coef,
 *                             cap_exp(x) = exp(min(x, floor(log(finfo(lp dtype).max) * 1e4) / 1e4)): no gradient
 *                             where the clamp is active
 *   AA_DPO_EXO_PAIR  sig(z) (logsig(z) - log(1 - e')) + sig(-z) (logsig(-z) - log e'), e' = e if e > 0 else 1e-3
 *   AA_DPO_DISCOPOP  -logsig(z) (1 - m) + exp(-z) m, m = sigmoid(z / discopop_tau)
 *   AA_DPO_AOT_PAIR  the kept pairs' a and, separately, their b sorted ascending (stable: NaN last, ties to the
 *                    smaller pair index); delta_k = a_(k) - b_(k); -(1-e) logsig(beta delta_k) - e logsig(-beta delta_k)
 *   AA_DPO_AOT       the same with pc - pr and rc - rr sorted in place of a and b
 * AOT: per_pair[0][i] is the loss at the sorted position of pair i's first key (a_i, or pc_i - pr_i), each row's
 * grad_seg entry the gradient at the position its key landed in; n_pairs <= AA_DPO_AOT_MAX_PAIRS.
 * label_smoothing is also legal for EXO_PAIR, AOT and AOT_PAIR.  exo_log_keep = log(1 - e') and exo_log_smooth =
 * log(e'): EXO's two constants, formed by the caller in double from its own label_smoothing (an fp32 copy of 0.1 is
 * not 0.1), both < 0; read by EXO_PAIR only.  f_alpha_coef (> 0, finite) must be 1 unless
 * f_divergence is ALPHA; discopop_tau (> 0, finite) must be 0.05 unless the type is DISCOPOP.  With f_divergence
 * REVERSE_KL and a type of aa_dpo_loss_obj the results are aa_dpo_loss_obj's, bit for bit.
 * ------------------------------------------------------------------------------------- */
enum {
  AA_DPO_EXO_PAIR = 8,
  AA_DPO_DISCOPOP = 9,
  AA_DPO_AOT = 10,
  AA_DPO_AOT_PAIR = 11,
  AA_DPO_AOT_MAX_PAIRS = 1024
};
enum { AA_DPO_FDIV_REVERSE_KL = 0, AA_DPO_FDIV_JS = 1, AA_DPO_FDIV_ALPHA = 2 };
int aa_dpo_loss_ext(const void *policy_lp, const void *ref_lp, int lp_dtype, int32_t n_pairs, int32_t width,
                    int64_t lp_row_stride, float scale_coeff, int mode, int loss_type, float label_smoothing,
                    float rpo_alpha, int f_divergence, float f_alpha_coef, float discopop_tau, float exo_log_keep,
                    float exo_log_smooth, const int32_t *counts,
                    const int64_t *input_ids, int32_t L, int64_t ids_row_stride, float *per_pair, float *grad_seg,
                    float *stats, uint32_t *counter, const int32_t *status, void *stream);

/* ---------------------------------------------------------------------------------------
 * Pair bookkeeping and slice sums of SimPO / ORPO / KTO (SURVEY.md 8f row 2).
 * aa_pair_slices: trainers/text_to_text/simpo.py:61-77 (orpo.py:61-77, kto.py:111-125): identical-pair test, last
 *   attended index of both rows, first index where the id rows differ -> out int32 [4][n_pairs] =
 *   valid, diverge_index, end_better, end_worse (bit-exact; 4 host syncs per pair in the reference).  Only a valid
 *   pair sets AA_STATUS_EMPTY_MASK / AA_STATUS_DIVERGE_RANGE: the reference skips an identical pair before it reads
 *   the masks.
 * aa_slice_sums: sums[r] = sum(lp[r, diverge : end + 1]) (simpo.py:78-79; Python slice semantics on the (2B, W)
 *   zero-padded log-prob rows), fp32 accumulate, rounded to the lp dtype in FAITHFUL mode; fp32 [2 * n_pairs] out.
 * The O(B) scalar formulas on top (log-ratio, log-sigmoid, odds ratio ...) are elementwise ATen ops on B-vectors in
 * the Python mirror -- bit-identical to the reference by construction; every O(rows * V) byte still goes through K1.
 * ------------------------------------------------------------------------------------- */
int aa_pair_slices(const int64_t *input_ids, int64_t ids_row_stride, const void *attention_mask, int mask_kind,
                   int64_t mask_row_stride, int32_t n_pairs, int32_t L, int32_t *out, int32_t *status, void *stream);
int aa_slice_sums(const void *lp, int lp_dtype, int64_t lp_row_stride, int32_t n_pairs, int32_t width,
                  const int32_t *slices, int mode, float *sums, void *stream);

/* ---------------------------------------------------------------------------------------
 * Reward-model pairwise loss (sibling of K2; SURVEY.md 8f row 2).  Replaces the loss tail of
 * trainers/text_to_text/rm.py:97-132: end_scores fp32 [2*n_pairs] (higher first, lower second) ->
 *   out[0] = mean(-logsigmoid(higher - lower)) + regularization * mean(square(all 2B scores)),
 *   out[1] = accuracy = mean(higher > lower);  grad_end_scores (optional) = d out[0] / d end_scores.
 * ------------------------------------------------------------------------------------- */
int aa_rm_pair_loss(const float *end_scores, int32_t n_pairs, float regularization, float *out,
                    float *grad_end_scores, void *stream);

/* ---------------------------------------------------------------------------------------
 * Cost-model pairwise loss (Safe RLHF's cost model; sibling of the RM loss).  Replaces the loss tail of
 * trainers/text_to_text/cost_model.py:97-144 (inherited by text_image_to_text/cost_model.py):
 *   end_scores [2*n_pairs] in score_dtype E (bf16 / f16 / f32; higher-cost rows first, lower second),
 *   better_signs / worse_signs [n_pairs]: is_better_safe / is_worse_safe cast to their product dtype with E
 *     (torch.result_type of the end scores and the sign tensor): E, or AA_F32 for float signs;
 *   loss   = scale_coeff * (-mean(logsigmoid(h * sb)) - mean(logsigmoid(l * sw))) - mean(logsigmoid(h - l))
 *            [+ regularization * mean(square(all 2B scores)) when regularization > 0],
 *            written as one element of dtype AA_F32 if either sign dtype is AA_F32, else E;
 *   stats  fp32 [2] = {loss, accuracy = mean(h > l)}  (the RM stats layout);
 *   grad_end_scores (optional) [2*n_pairs] in E = d loss / d end_scores.
 * FAITHFUL rounds where the eager ops round, and the gradient restates autograd's chain and casts;
 * AA_MODE_F32 keeps fp32 throughout and rounds the loss and the gradient once (stats[0] keeps the fp32 loss).
 * One CTA.
 * ------------------------------------------------------------------------------------- */
int aa_cost_pair_loss(const void *end_scores, int score_dtype, const void *better_signs, int better_dtype,
                      const void *worse_signs, int worse_dtype, int32_t n_pairs, float scale_coeff,
                      float regularization, int mode, void *loss, float *stats, void *grad_end_scores, void *stream);

/* ---------------------------------------------------------------------------------------
 * K3  scalar score head of the reward / critic models: scores[r] = <hidden[r,:], w>.
 * Replaces `self.score_head(last_hidden_state)` (models/llama.py:62-63, opt.py, llava.py:62-63,
 * qwen2_vl.py:59-60, qwen2_audio.py:77-78).  FAITHFUL: fp32 dot rounded to the hidden dtype
 * (what nn.Linear returns) and then widened if out_dtype is AA_F32 (`.float()`).
 * A GEMV (N = 1): HBM-bound on reading hidden, H * sizeof per row.
 * ------------------------------------------------------------------------------------- */
int aa_score_head_fwd(const void *hidden, int dtype, int64_t n_rows, int32_t H, int64_t row_stride,
                      const void *weight, void *scores, int out_dtype, int mode, void *stream);

/* end_index = last nonzero of each attention-mask row (models/llama.py:71 `m.nonzero()[-1]`),
 * or L-1 when mask == NULL (llava.py:64-66 / qwen2_vl.py:62-64 take position -1);
 * end_scores[b] = scores[b, end_index[b]] (fp32); optional end_hidden (B, H) gather. */
int aa_score_end(const void *scores, int scores_dtype, int64_t scores_row_stride,
                 const void *mask, int mask_kind, int64_t mask_row_stride, int32_t B, int32_t L,
                 int64_t *end_index, float *end_scores,
                 const void *hidden, int hidden_dtype, int64_t hidden_batch_stride,
                 int64_t hidden_row_stride, int32_t H, void *end_hidden,
                 int32_t *status, void *stream);

/* Backward of the head: grad_hidden[r,:] = g[r] * w  (dtype of hidden), and
 * grad_weight[:] = sum_r g[r] * hidden[r,:] (fp32, deterministic two-stage reduction through
 * `partial` = fp32 [n_partials][H] scratch; n_partials = value returned in *n_partials_needed
 * when partial == NULL). */
int aa_score_head_bwd(const void *hidden, int dtype, int64_t n_rows, int32_t H, int64_t row_stride,
                      const void *weight, const void *grad_scores, int grad_dtype,
                      void *grad_hidden, int64_t grad_row_stride, float *grad_weight,
                      float *partial, int32_t *n_partials_needed, int mode, void *stream);

/* ---------------------------------------------------------------------------------------
 * K4  PPO preparation, one launch: KL-shaped rewards, GAE reverse scan, returns.
 * Replaces trainers/text_to_text/ppo.py:528-547 (add_kl_divergence_regularization) and
 * :487-508 (get_advantages_and_returns) -- a Python loop over t in the reference -- plus the
 * row sums behind the kl_divergence / reward_with_kl_penalty / generated-length metrics
 * (:361-369).  All 2-D inputs are (B, W) with their own row strides; mask is torch.bool.
 *   old_rewards : (B, W) lp dtype (FAITHFUL) or fp32
 *   advantages, returns : (B, W - start), `adv_dtype` (torch promotion of values x rewards)
 *   row_stats : fp32 [B][8] = kl_sum, reward_kl_sum, mask_count(start..), adv_row_mean,
 *               ret_row_mean, end_index, 0, 0
 * log_probs == ref_log_probs == reward == NULL: GAE only -- `old_rewards` is then an INPUT holding
 * precomputed per-token rewards (PPOTrainer.get_advantages_and_returns called on its own).
 * The scan is a warp-shuffle affine scan (A_t = d_t + gamma*lambda*A_{t+1}) in fp32; when
 * adv_dtype is 16-bit in FAITHFUL mode the recurrence is evaluated sequentially with the
 * reference's per-op rounding so that results are reproducible bit for bit.
 * ------------------------------------------------------------------------------------- */
int aa_ppo_prep(const void *log_probs, const void *ref_log_probs, int lp_dtype, int64_t lp_row_stride,
                const float *reward, const void *values, int val_dtype, int64_t val_row_stride,
                const uint8_t *mask, int64_t mask_row_stride, int32_t B, int32_t W, int32_t start,
                float kl_coeff, float clip_range_score, float gamma, float gae_lambda, int mode,
                void *old_rewards, int rew_dtype, void *advantages, void *returns, int adv_dtype,
                float *row_stats, int32_t *status, void *stream);
/* KL estimators of the per-token penalty (aa_ppo_prep_kl) and of GRPO's per-token loss (aa_grpo_loss_kl,
 * aa_logprob_grpo_fused_kl), with d = lp - ref:  K1 d ;  K2 0.5 * d^2 ;  K3 exp(-d) + d - 1 (each op rounded as the
 * eager expression in ops.KL_ESTIMATORS rounds it). */
enum { AA_KL_K1 = 0, AA_KL_K2 = 1, AA_KL_K3 = 2 };
/* aa_ppo_prep with the penalty reward -kl_coeff * KL taken by `kl_estimator`; row_stats[b][0] stays the k1 row sum
 * (the kl_divergence metric).  kl_coeff must be finite.  With AA_KL_K1 the outputs are bit-identical to aa_ppo_prep;
 * the GAE-only form (NULL log-probs) is aa_ppo_prep's. */
int aa_ppo_prep_kl(const void *log_probs, const void *ref_log_probs, int lp_dtype, int64_t lp_row_stride,
                   const float *reward, const void *values, int val_dtype, int64_t val_row_stride,
                   const uint8_t *mask, int64_t mask_row_stride, int32_t B, int32_t W, int32_t start,
                   float kl_coeff, int kl_estimator, float clip_range_score, float gamma, float gae_lambda, int mode,
                   void *old_rewards, int rew_dtype, void *advantages, void *returns, int adv_dtype,
                   float *row_stats, int32_t *status, void *stream);

/* ---------------------------------------------------------------------------------------
 * K4r  Multi-PPO returns, one launch: trainers/text_to_text/multi_ppo.py:510-591
 * (get_advantages_and_returns + cumulative_returns, a Python loop over t in the reference) for
 * the four non-GAE estimators.  `rewards` is K4's (B, W) `old_rewards` (row stride in elements),
 * mask is torch.bool (B, W).  The group estimators reshape the flattened (B, W) token rewards to
 * (-1, n): a group is n consecutive flat elements, possibly spanning rows (SURVEY.md H9), so
 * B * W must be a multiple of n.  The carry c = r_t + gamma * c is float32; each c is stored
 * rounded to the rewards dtype (FAITHFUL) and, with mask_outputs != 0, multiplied by the mask
 * (get_advantages_and_returns; mask_outputs == 0 is cumulative_returns on its own).
 *   advantages, returns : (B, W - start) contiguous, `out_dtype` (equal tensors; separate buffers)
 *   row_stats           : optional fp32 [B][8] in K4's layout; lanes 3 and 4 are overwritten with
 *                         the masked row means of advantages and returns, the rest is untouched
 * ------------------------------------------------------------------------------------- */
enum { AA_EST_REINFORCE = 0, AA_EST_RLOO = 1, AA_EST_REINFORCE_BASELINE = 2, AA_EST_GROUP_NORM = 3 };
int aa_ppo_returns(const void *rewards, int rew_dtype, int64_t rew_row_stride, const uint8_t *mask,
                   int64_t mask_row_stride, int32_t B, int32_t W, int32_t start, int estimator,
                   int32_t n_samples_per_prompt, float gamma, int mode, int mask_outputs, void *advantages,
                   void *returns, int out_dtype, float *row_stats, void *stream);

/* ---------------------------------------------------------------------------------------
 * Advantage whitening over a rollout: TRL's / verl's masked_whiten(A, m, shift_mean=True) over the advantages A
 * and the actor-loss mask m of EVERY micro-batch of one rollout (and every data-parallel rank):
 *   n = sum m,  mean = sum m A / n,  var = sum m (A - mean)^2 / (n - 1),
 *   A' = (A - mean) * rsqrt(var + 1e-8) where m, 0 where not m.
 * The statistics are fp64; mean and rstd are formed once in fp64 and rounded to fp32; (A - mean) * rstd is fp32,
 * rounded once to the advantages' dtype.  Every sum has a fixed order (no floating-point atomics): a run gives the
 * same bits every time.  For K micro-batches:
 *   aa_whiten_moments x K : micro-batch k's (B, W) advantages (bf16 / f16 / f32, row stride in elements) and
 *                           torch.bool mask -> its fp64 (n, sum A, sum A^2) in moments[3k .. 3k + 2] of a
 *                           caller-owned (K, 3) buffer (one CTA per launch)
 *   aa_whiten_reduce      : total (3,) = the K slots summed in slot order; across ranks the caller all-reduces
 *                           (SUM) this fixed-size triple before the applies
 *   aa_whiten_apply x K   : rewrites micro-batch k's advantages in place from `total`.  n < 2 sets
 *                           AA_STATUS_WHITEN_COUNT in `status` and leaves the advantages unchanged.
 * ------------------------------------------------------------------------------------- */
int aa_whiten_moments(const void *advantages, int adv_dtype, int64_t adv_row_stride, const uint8_t *mask,
                      int64_t mask_row_stride, int32_t B, int32_t W, double *moments, int32_t k, int32_t K,
                      void *stream);
int aa_whiten_reduce(const double *moments, int32_t K, double *total, void *stream);
int aa_whiten_apply(void *advantages, int adv_dtype, int64_t adv_row_stride, const uint8_t *mask,
                    int64_t mask_row_stride, int32_t B, int32_t W, const double *total, int32_t *status, void *stream);

/* ---------------------------------------------------------------------------------------
 * K5  PPO losses, forward AND backward in one launch each (the backward is elementwise).
 * actor : trainers/text_to_text/ppo.py:291-307  (+ utils/tools.py:460-467 masked_mean)
 * critic: trainers/text_to_text/ppo.py:510-526
 * Inputs are (B, Wm) views (caller passes pointers already offset to column `start`).
 *   loss      : fp32 [2]: [0] = the loss; when the promoted dtype of the inputs is 16-bit, the first two bytes of [1]
 *               hold the same value in that dtype (the caller views it as the 0-dim bf16 / f16 tensor the reference's
 *               loss is: no conversion launch)
 *   grad      : (B, Wm) d loss / d new_log_probs (resp. new values), input dtype, or NULL
 *   value_tail_lens / value_src_width (critic, optional): `values` is then the RAW (B, value_src_width) tensor
 *               `scores.squeeze(-1)[:, :-1]` and the kernel reads values[b, t] = t < R_b ? raw[b, value_src_width - R_b + t] : 0
 *               with R_b = clamp(value_tail_lens[b], 0, value_src_width) (the pad_sequence of per-sample tails of
 *               text_image_to_text/ppo.py:318-330 folded into the load); aa_tail_scatter_scaled is its exact transpose.
 *   row_mean  : optional fp32 [B], masked row mean of `new` values (critic: reward_value metric)
 *   counter   : device uint32 scratch (zero before first use; self-cleaning)
 * ------------------------------------------------------------------------------------- */
int aa_ppo_actor_loss(const void *log_probs, int64_t lp_stride, const void *old_log_probs,
                      int64_t old_stride, int lp_dtype, const void *advantages, int64_t adv_stride,
                      int adv_dtype, const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t Wm,
                      float clip_range_ratio, int mode, float *loss, void *grad, int64_t grad_stride,
                      float *row_scratch, uint32_t *counter, void *stream);

/* aa_ppo_actor_loss with the objective's options (ops.ActorObjective):
 *   clip_low / clip_high : the ratio is clamped to [1 - clip_low, 1 + clip_high] (clip-higher: clip_high > clip_low);
 *                          0 <= clip_low < 1, clip_high >= 0
 *   dual_clip            : 0 (off) or c > 1: for adv < 0 the objective is max(min(s1, s2), c * adv)
 *   loss_agg             : AA_AGG_SEQ_MEAN_TOKEN_MEAN (the reference's masked_mean) or AA_AGG_TOKEN_MEAN
 *                          (-(s * mask).sum() / mask.sum() over the whole micro-batch)
 *   clip_frac            : optional fp32[2]: [0] the masked-in share of tokens whose clipped branch is strictly smaller,
 *                          [1] the share of masked-in adv < 0 tokens where c * adv wins (0 without such tokens), both
 *                          aggregated like the loss
 *   row_scratch          : fp32 [4 * B]
 * With clip_low == clip_high == clip_range_ratio, dual_clip 0 and AA_AGG_SEQ_MEAN_TOKEN_MEAN the loss and gradient
 * are bit-identical to aa_ppo_actor_loss.  Arguments are checked before any CUDA call. */
/* AA_AGG_SEQ_MEAN_TOKEN_SUM_NORM (Dr. GRPO: sum(loss * mask) / (B * K)) is taken by the GRPO objective entry points only. */
enum { AA_AGG_SEQ_MEAN_TOKEN_MEAN = 0, AA_AGG_TOKEN_MEAN = 1, AA_AGG_SEQ_MEAN_TOKEN_SUM_NORM = 2 };
int aa_ppo_actor_loss_obj(const void *log_probs, int64_t lp_stride, const void *old_log_probs, int64_t old_stride,
                          int lp_dtype, const void *advantages, int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                          int64_t mask_stride, int32_t B, int32_t Wm, float clip_low, float clip_high, float dual_clip,
                          int loss_agg, int mode, float *loss, void *grad, int64_t grad_stride, float *clip_frac,
                          float *row_scratch, uint32_t *counter, void *stream);

/* aa_ppo_actor_loss_obj with a KL loss term: the actor minimises  loss + kl_loss_coeff * agg(KL, mask), KL the
 * per-token estimate (AA_KL_*, kl_estimator) of log_probs against ref_log_probs (lp_dtype, (B, Wm) with row stride
 * ref_stride), agg the objective's aggregation over the same mask.
 *   loss      : the clipped objective alone, as aa_ppo_actor_loss_obj writes it
 *   kl_loss   : fp32 [1], agg(KL) without the coefficient (in the log-probs' dtype's rounding in FAITHFUL mode)
 *   grad      : d (loss + kl_loss_coeff * agg(KL)) / d log_probs
 *   row_scratch: fp32 [5 * B]
 * kl_loss_coeff must be finite and > 0 and ref_log_probs non-NULL; these and the objective's checks run before any
 * CUDA call. */
int aa_ppo_actor_loss_kl(const void *log_probs, int64_t lp_stride, const void *old_log_probs, int64_t old_stride,
                         int lp_dtype, const void *advantages, int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                         int64_t mask_stride, int32_t B, int32_t Wm, float clip_low, float clip_high, float dual_clip,
                         int loss_agg, int mode, const void *ref_log_probs, int64_t ref_stride, float kl_loss_coeff,
                         int kl_estimator, float *loss, float *kl_loss, void *grad, int64_t grad_stride,
                         float *clip_frac, float *row_scratch, uint32_t *counter, void *stream);

int aa_ppo_critic_loss(const void *values, int64_t val_stride, const void *old_values,
                       int64_t old_stride, int val_dtype, const void *returns, int64_t ret_stride,
                       int ret_dtype, const uint8_t *mask, int64_t mask_stride, int32_t B, int32_t Wm,
                       float clip_range_value, int mode, float *loss, void *grad, int64_t grad_stride,
                       float *row_mean, float *row_scratch, uint32_t *counter, const int32_t *value_tail_lens,
                       int32_t value_src_width, void *stream);

/* Adjoint of the tail gather above times an upstream scalar, one launch for the whole (B, out_width) tile (zeros
 * included).  With the same R_b = clamp(lens[b], 0, src_width) and n_b = min(R_b, W):
 * out[b, t] = src_width - R_b <= t < src_width - R_b + n_b ? scale * grad[b, t - (src_width - R_b)] : 0.  grad (B, W) and out
 * share `dtype`; scale: optional device scalar of scale_dtype (fp32 product, rounded once).  Replaces the autograd of
 * `scores.squeeze(-1)[:, :-1]` + per-sample slicing + pad_sequence (SliceBackward / CatBackward / a zero-filled tile). */
int aa_tail_scatter_scaled(const void *grad, int dtype, int64_t grad_row_stride, const int32_t *lens, int32_t B, int32_t W,
                           int32_t src_width, const void *scale, int scale_dtype, void *out, int64_t out_row_stride,
                           int32_t out_width, void *stream);

/* ---------------------------------------------------------------------------------------
 * K1f  The actor half of a PPO rl_step in ONE pass over the logits tile: log-probs of the response tails
 * (K1), d actor_loss / d log-prob per token (K5's arithmetic) and the gradient tile (K1b) -- the clipped-ratio
 * objective is a masked mean of per-token terms, so a row's gradient only needs that row's own log-prob plus values
 * known before the forward.  Each scored row is streamed twice by the same CTA (the second pass is served by the
 * 126 MB L2), so HBM sees V*e read + V*e written per scored row instead of 2*V*e + V*e.
 * Replaces trainers/text_image_to_text/ppo.py:296-316 (text: trainers/text_to_text/ppo.py:336-349):
 * actor forward logits -> gather_log_probabilities -> actor_loss_fn -> backward up to d logits.
 *   row plan    : as aa_logprob_bwd in tile mode (segments = samples, n_tile_rows / n_segments tile rows each;
 *                 host RowPlan or aa_tail_plan_build table)
 *   log_probs   : (n_segments, W) lp_dtype, zero-initialised by the caller (pad columns stay 0)
 *   stat_*      : optional fp32 [n scored rows] (max, logsum) as aa_logprob_fwd
 *   old_log_probs (lp_dtype) / advantages / mask : (n_segments, W) with element row strides
 *   grad_logits : every tile row is written (scored rows: d loss / d logits for an upstream gradient of 1; others 0)
 *   row_scratch : device scratch, 48 bytes per tile row, 16-byte aligned
 * The loss VALUE is aa_ppo_actor_loss on `log_probs`; aa_scale_tile applies an upstream scalar != 1. */
int aa_logprob_actor_fused(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                           const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                           const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                           const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                           float *stat_max, float *stat_logsum, const void *old_log_probs, int64_t old_stride,
                           const void *advantages, int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                           int64_t mask_stride, int32_t W, float clip_range_ratio, int mode, void *grad_logits,
                           int64_t grad_row_stride, void *row_scratch, int32_t *status, void *stream);
/* aa_logprob_actor_fused for the regularised objective  actor_loss - entropy_coeff * masked_mean(H, mask): the
 * entropy of every scored row is written to `entropy` (fp32, laid out like log_probs, zero-initialised by the caller)
 * and the gradient tile carries the entropy's gradient (aa_logprob_bwd_entropy's formula) with
 * g_H = -entropy_coeff * mask / (n_segments * mask count of the row).  log_probs, stat_* and the rows with g_H == 0
 * are bit-identical to aa_logprob_actor_fused.  row_scratch: 48 bytes per tile row plus 4 bytes per segment. */
int aa_logprob_actor_fused_entropy(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                   const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                   const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                                   const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                                   float *stat_max, float *stat_logsum, const void *old_log_probs, int64_t old_stride,
                                   const void *advantages, int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                                   int64_t mask_stride, int32_t W, float clip_range_ratio, int mode, void *grad_logits,
                                   int64_t grad_row_stride, void *row_scratch, int32_t *status, float entropy_coeff,
                                   float *entropy, void *stream);
/* aa_logprob_actor_fused / _entropy with the objective of aa_ppo_actor_loss_obj (clip_low, clip_high, dual_clip,
 * loss_agg: same meaning and checks).  entropy == NULL: the plain kernel; otherwise the entropy-bonus kernel of
 * aa_logprob_actor_fused_entropy, whose g_H under AA_AGG_TOKEN_MEAN is -entropy_coeff / (masked-in tokens of the
 * micro-batch) on every masked-in token.  Under AA_AGG_TOKEN_MEAN every row's coefficient is -1 / that count.  With the
 * default objective the outputs are bit-identical to aa_logprob_actor_fused / _entropy.  row_scratch: 48 bytes per
 * tile row plus 4 bytes per segment. */
int aa_logprob_actor_fused_obj(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                               const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                               const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                               const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                               float *stat_max, float *stat_logsum, const void *old_log_probs, int64_t old_stride,
                               const void *advantages, int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                               int64_t mask_stride, int32_t W, float clip_low, float clip_high, float dual_clip,
                               int loss_agg, int mode, void *grad_logits, int64_t grad_row_stride, void *row_scratch,
                               int32_t *status, float entropy_coeff, float *entropy, void *stream);

/* aa_logprob_actor_fused_obj with the KL loss term of aa_ppo_actor_loss_kl: the gradient tile carries
 * d (actor_loss + kl_loss_coeff * agg(KL, mask)) / d logits.  ref_log_probs (lp_dtype) is laid out like log_probs
 * (contiguous (n_segments, W)) and is read at each log-prob's own index.  log_probs, stat_* and entropy are
 * bit-identical to aa_logprob_actor_fused_obj; the loss value and agg(KL) are aa_ppo_actor_loss_kl's on log_probs.
 * row_scratch: 48 bytes per tile row plus 8 bytes per segment.  kl_loss_coeff must be finite and > 0 and
 * ref_log_probs non-NULL; these and the objective's checks run before any CUDA call. */
int aa_logprob_actor_fused_kl(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                              const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                              const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                              const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                              float *stat_max, float *stat_logsum, const void *old_log_probs, int64_t old_stride,
                              const void *advantages, int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                              int64_t mask_stride, int32_t W, float clip_low, float clip_high, float dual_clip,
                              int loss_agg, int mode, void *grad_logits, int64_t grad_row_stride, void *row_scratch,
                              int32_t *status, float entropy_coeff, float *entropy, const void *ref_log_probs,
                              float kl_loss_coeff, int kl_estimator, void *stream);

/* The same single pass for the mean cross-entropy behind `outputs.loss` (trainers/text_to_text/sft.py:95-98
 * `SupervisedTrainer.loss`, ppo.py:400-408 `ptx_step`; transformers' ForCausalLMLoss): every row whose label !=
 * ignore_index has the upstream gradient -loss_scale / n_valid, known before the row is read, so the fp32 log-probs
 * AND d (loss_scale * loss) / d logits come out of one pass over the valid rows (HBM: V*e read + V*e written per valid
 * row; aa_logprob_fwd + aa_logprob_bwd: 2*V*e + V*e).  Ignored rows cost no reads (log-prob 0, zero gradient row).
 *   labels      : the SHIFTED labels the row plan addresses; n_labels = how many of them to count for n_valid
 *   log_probs   : fp32, zero-initialised by the caller; the loss value is aa_nll_mean over it
 *   row_scratch : 48 bytes per tile row (16-byte aligned); coeff_scratch: one device float */
int aa_logprob_ce_fused(const void *logits, int logits_dtype, int64_t row_stride, int32_t V, const int64_t *labels,
                        int64_t n_labels, int64_t ignore_index, int32_t n_segments, const int64_t *seg_logit_off,
                        const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                        const int64_t *seg_tile_row, int64_t n_tile_rows, float *log_probs, float loss_scale,
                        void *grad_logits, int64_t grad_row_stride, void *row_scratch, float *coeff_scratch,
                        int32_t *status, void *stream);

/* ... and for the GRPO loss (trainers/text_to_text/grpo.py:290-312): per-token loss -(exp(lp - lp.detach()) * A - beta * KL)
 * with the k3 KL against the reference log-probs, counted up to and including the first eos of each completion, token
 * mean.  d loss / d lp of a token needs its own log-prob, the reference model's log-prob (scored BEFORE this call) and
 * the sequence's group advantage.  Segments = sequences; log_probs (n_segments, K) lp_dtype zero-initialised by the
 * caller; ref_log_probs (n_segments, K) lp_dtype; advantages fp32 [n_segments]; completion_tokens (n_segments, K).
 * row_end (int32 [n_segments]) and total (fp32 [1]) are outputs of the mask pass; the loss VALUE is aa_grpo_loss on
 * `log_probs`.  counter: device uint32 scratch (zero before first use; self-cleaning). */
int aa_logprob_grpo_fused(const void *logits, int logits_dtype, int64_t row_stride, int32_t V, const int64_t *labels,
                          int32_t n_segments, const int64_t *seg_logit_off, const int64_t *seg_label_off,
                          const int64_t *seg_out_off, const int64_t *seg_cum, const int64_t *seg_tile_row,
                          int64_t n_tile_rows, void *log_probs, int lp_dtype, const void *ref_log_probs, int64_t ref_stride,
                          const float *advantages, const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id,
                          int32_t K, float beta, int mode, void *grad_logits, int64_t grad_row_stride, void *row_scratch,
                          int32_t *row_end, float *total, uint32_t *counter, int32_t *status, void *stream);
/* The same launch with the entropy of every scored row (fp32, aa_logprob_fwd_entropy's definition) written to entropy,
 * laid out like log_probs ((n_segments, K), zero-initialised by the caller), from the (max, sum-exp) pass (phase A).
 * log_probs, the gradient tile and everything else are bit-identical to aa_logprob_grpo_fused. */
int aa_logprob_grpo_fused_entropy(const void *logits, int logits_dtype, int64_t row_stride, int32_t V, const int64_t *labels,
                                  int32_t n_segments, const int64_t *seg_logit_off, const int64_t *seg_label_off,
                                  const int64_t *seg_out_off, const int64_t *seg_cum, const int64_t *seg_tile_row,
                                  int64_t n_tile_rows, void *log_probs, int lp_dtype, const void *ref_log_probs,
                                  int64_t ref_stride, const float *advantages, const int64_t *completion_tokens,
                                  int64_t tok_stride, int64_t eos_id, int32_t K, float beta, int mode, void *grad_logits,
                                  int64_t grad_row_stride, void *row_scratch, int32_t *row_end, float *total,
                                  uint32_t *counter, int32_t *status, float *entropy, void *stream);
/* aa_logprob_grpo_fused_entropy for  loss - entropy_coeff * (H * mask).sum() / mask.sum()  over the completion mask:
 * the tile also carries the entropy's gradient (aa_logprob_bwd_entropy's formula) with g_H = -entropy_coeff / total for
 * counted tokens.  log_probs, row_end, total and the rows with g_H == 0 are bit-identical to aa_logprob_grpo_fused. */
int aa_logprob_grpo_fused_entropy_grad(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                                       const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                                       const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                                       const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                                       const void *ref_log_probs, int64_t ref_stride, const float *advantages,
                                       const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t K,
                                       float beta, int mode, void *grad_logits, int64_t grad_row_stride,
                                       void *row_scratch, int32_t *row_end, float *total, uint32_t *counter,
                                       int32_t *status, float *entropy, float entropy_coeff, void *stream);
/* aa_logprob_grpo_fused with GRPO's clipped objective (aa_grpo_loss_obj's per-token loss and aggregation; clip_low,
 * clip_high, dual_clip, loss_agg: same meaning and checks).  old_log_probs: NULL (the ratio is exp(lp - lp) = 1: the
 * first update of a rollout) or the rollout-time policy log-probs (lp_dtype, laid out exactly like log_probs: read at
 * the log-prob's own index).  entropy == NULL: the plain kernel; otherwise entropy is written as by
 * aa_logprob_grpo_fused_entropy and, with entropy_coeff != 0, the tile carries the bonus's gradient with
 * g_H = -entropy_coeff / total (a token mean over the completion mask under every aggregation).  The loss VALUE and the
 * clip fractions are aa_grpo_loss_obj on `log_probs`. */
int aa_logprob_grpo_fused_obj(const void *logits, int logits_dtype, int64_t row_stride, int32_t V, const int64_t *labels,
                              int32_t n_segments, const int64_t *seg_logit_off, const int64_t *seg_label_off,
                              const int64_t *seg_out_off, const int64_t *seg_cum, const int64_t *seg_tile_row,
                              int64_t n_tile_rows, void *log_probs, int lp_dtype, const void *ref_log_probs,
                              int64_t ref_stride, const void *old_log_probs, const float *advantages,
                              const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t K, float beta,
                              float clip_low, float clip_high, float dual_clip, int loss_agg, int mode, void *grad_logits,
                              int64_t grad_row_stride, void *row_scratch, int32_t *row_end, float *total,
                              uint32_t *counter, int32_t *status, float *entropy, float entropy_coeff, void *stream);
/* aa_logprob_grpo_fused_obj with the per-token KL taken by `kl_estimator` (AA_KL_*): the loss value and clip fractions
 * are then aa_grpo_loss_kl's.  With AA_KL_K3 every output is bit-identical to aa_logprob_grpo_fused_obj. */
int aa_logprob_grpo_fused_kl(const void *logits, int logits_dtype, int64_t row_stride, int32_t V, const int64_t *labels,
                             int32_t n_segments, const int64_t *seg_logit_off, const int64_t *seg_label_off,
                             const int64_t *seg_out_off, const int64_t *seg_cum, const int64_t *seg_tile_row,
                             int64_t n_tile_rows, void *log_probs, int lp_dtype, const void *ref_log_probs,
                             int64_t ref_stride, const void *old_log_probs, const float *advantages,
                             const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t K, float beta,
                             float clip_low, float clip_high, float dual_clip, int loss_agg, int kl_estimator, int mode,
                             void *grad_logits, int64_t grad_row_stride, void *row_scratch, int32_t *row_end,
                             float *total, uint32_t *counter, int32_t *status, float *entropy, float entropy_coeff,
                             void *stream);

/* tile[0..n) *= *scale unless *scale == 1 (checked on the device: the usual `loss.backward()` costs one empty launch).
 * Contiguous tile; scale: device scalar of scale_dtype.  The autograd backward of the K1f node. */
int aa_scale_tile(void *tile, int dtype, int64_t n, const void *scale, int scale_dtype, void *stream);

/* ---------------------------------------------------------------------------------------
 * Mean negative log-likelihood over the rows whose label != ignore_index: the epilogue that turns
 * K1's per-token log-probs into the causal-LM cross-entropy behind `outputs.loss`
 * (trainers/text_to_text/sft.py:95-98 `SupervisedTrainer.loss`, ppo.py:400-408 `ptx_step`;
 * transformers' ForCausalLMLoss: fp32 log-softmax, mean over non-ignored tokens).
 *   loss[0] = -sum(logp[valid]) / n_valid ; neg_inv_count[0] = -1 / n_valid (the per-row upstream
 *   gradient that aa_logprob_bwd takes as grad_scale).  partial: fp32 [2 * 256] scratch.
 * ------------------------------------------------------------------------------------- */
int aa_nll_mean(const void *logp, int dtype, const int64_t *labels, int64_t n, int64_t ignore_index,
                float *loss, float *neg_inv_count, float *partial, uint32_t *counter, void *stream);

/* ---------------------------------------------------------------------------------------
 * GRPO (sibling of K5; SURVEY.md 8f row 2).  trainers/text_to_text/grpo.py:268-318.
 * aa_group_advantages: rewards fp32 [n_groups][group_size] -> (r - mean) / (std_unbiased + 1e-4)   (:268-274)
 * aa_grpo_loss: per-token KL exp(ref - lp) - (ref - lp) - 1, per-token loss -(A - beta * KL), completion mask up to
 *   and including the first eos of `completion_tokens` (B, K), loss = sum(masked) / sum(mask)      (:290-312),
 *   forward AND d loss / d log_probs (lp dtype; NULL to skip) in two launches.
 *   row_end: int32 [B] scratch (out: counted tokens per row); scratch: fp32 [1 + B]; counter: uint32 [2], zeroed once.
 * ------------------------------------------------------------------------------------- */
int aa_group_advantages(const float *rewards, int32_t n_groups, int32_t group_size, float *advantages, void *stream);
int aa_grpo_loss(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride, int lp_dtype,
                 const float *advantages, const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id,
                 int32_t B, int32_t K, float beta, int mode, float *loss, void *grad, int64_t grad_stride,
                 int32_t *row_end, float *scratch, uint32_t *counter, void *stream);
/* Dr. GRPO's advantages: r - group mean, no std scaling (the group mean as aa_group_advantages computes it). */
int aa_group_advantages_centered(const float *rewards, int32_t n_groups, int32_t group_size, float *advantages,
                                 void *stream);
/* aa_grpo_loss with GRPO's clipped objective.  With r = exp(lp - old):
 *   s = min(A * r, A * clamp(r, 1 - clip_low, 1 + clip_high)); dual_clip c > 1 (0 = off): s = max(s, c * A) where A < 0;
 *   per-token loss = -(s - beta * KL)  (the KL of aa_grpo_loss);
 *   loss_agg: AA_AGG_TOKEN_MEAN  sum(loss * mask) / sum(mask)  (aa_grpo_loss's aggregation),
 *             AA_AGG_SEQ_MEAN_TOKEN_MEAN  the mean over rows of each row's token mean,
 *             AA_AGG_SEQ_MEAN_TOKEN_SUM_NORM  sum(loss * mask) / (B * K).
 *   old_log_probs: lp_dtype with row stride old_stride, or NULL for the log-probs themselves (r == 1).
 *   clip_frac: optional fp32[2] as aa_ppo_actor_loss_obj's (seq-mean-token-mean: mean of the row fractions; the other
 *              two aggregations: token fractions over the completion mask).
 * Arguments are checked before any CUDA call; scratch: fp32 [1 + 4 * B]; counter: uint32 [2], zeroed once. */
int aa_grpo_loss_obj(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                     const void *old_log_probs, int64_t old_stride, int lp_dtype, const float *advantages,
                     const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B, int32_t K,
                     float beta, float clip_low, float clip_high, float dual_clip, int loss_agg, int mode, float *loss,
                     void *grad, int64_t grad_stride, float *clip_frac, int32_t *row_end, float *scratch,
                     uint32_t *counter, void *stream);
/* aa_grpo_loss_obj with the per-token KL taken by `kl_estimator` (AA_KL_*, below) instead of k3; with AA_KL_K3 the
 * outputs are bit-identical to aa_grpo_loss_obj.  An unknown estimator code is refused before any CUDA call. */
int aa_grpo_loss_kl(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                    const void *old_log_probs, int64_t old_stride, int lp_dtype, const float *advantages,
                    const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B, int32_t K,
                    float beta, float clip_low, float clip_high, float dual_clip, int loss_agg, int kl_estimator,
                    int mode, float *loss, void *grad, int64_t grad_stride, float *clip_frac, int32_t *row_end,
                    float *scratch, uint32_t *counter, void *stream);
/* aa_grpo_loss_kl with GSPO's sequence-level ratio (Zheng et al. 2025; TRL's importance_sampling_level="sequence"):
 * one ratio per row, w = exp(S / n), with S = sum(((lp - old) * mask)) rounded once to lp_dtype and n the row's token
 * count; w, the clip bounds and s = min(A * w, A * clamp(w, 1 - clip_low, 1 + clip_high)) (and dual-clip) are fp32 in
 * both modes.  The per-token KL, the aggregations and the clip fractions are aa_grpo_loss_kl's; every counted token of
 * a row shares w, so the fractions count clipped sequences (seq-mean-token-mean) or the tokens in them.  Each token's
 * gradient through the ratio is d loss / d w * w / n, cast once to the gradient's rounding dtype.  old_log_probs is
 * required (without it w == 1 and the objective is aa_grpo_loss_kl's at ratio 1).  Arguments are checked before any
 * CUDA call. */
int aa_grpo_loss_seq(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                     const void *old_log_probs, int64_t old_stride, int lp_dtype, const float *advantages,
                     const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B, int32_t K,
                     float beta, float clip_low, float clip_high, float dual_clip, int loss_agg, int kl_estimator,
                     int mode, float *loss, void *grad, int64_t grad_stride, float *clip_frac, int32_t *row_end,
                     float *scratch, uint32_t *counter, void *stream);
/* aa_grpo_loss_seq's objective (sequence 1) or aa_grpo_loss_kl's (sequence 0; old_log_probs may then be NULL: ratio
 * 1) under the top-entropy mask (Wang et al. 2025; TRL's top_entropy_quantile): a counted token with
 * entropy[b * ent_stride + t] < thr[0] (fp32, e.g. from aa_entropy_select_lo; NaN keeps nothing) has the per-token loss
 * -(s * 0 - beta * KL), so s sends it no gradient.  At sequence level s's gradient reaches the row's ratio from the
 * kept tokens only, and through the ratio every counted token's log-prob, as autograd of the masked loss gives it.
 * The KL term, the aggregation's denominators and the clip fractions are the unmasked ones.  Arguments are checked
 * before any CUDA call. */
int aa_grpo_loss_topent(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                        const void *old_log_probs, int64_t old_stride, int lp_dtype, const float *advantages,
                        const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B, int32_t K,
                        float beta, float clip_low, float clip_high, float dual_clip, int loss_agg, int kl_estimator,
                        int sequence, int mode, float *loss, void *grad, int64_t grad_stride, float *clip_frac,
                        const float *entropy, int64_t ent_stride, const float *thr, int32_t *row_end, float *scratch,
                        uint32_t *counter, void *stream);

/* Top-entropy threshold: thr = torch.quantile(H[counted], q) (linear interpolation) over every counted token of every
 * rank, as an exact radix select on order-preserving keys, with no host sync.
 *   aa_grpo_row_end      : GRPO's completion mask pass alone (row_end[b] = tokens up to and including the first eos,
 *                          total[0] = their fp32 count), the rule aa_grpo_loss* apply.
 *   aa_entropy_hist_hi   : hist (uint32[65537], zeroed here) = counts of the high 16 bits of the counted entropies' keys,
 *                          hist[65536] = their NaNs.  counted: t < row_end[b], or mask[b * mask_stride + t] != 0 (give
 *                          exactly one); entropy fp32 (B, K), row stride ent_stride.  B * K < 2^31.
 *   (across ranks the caller all-reduces hist with SUM)
 *   aa_entropy_select_hi : one block; sel (uint32[8]) = the count N, the NaN count, and for lo = floor(rank) and
 *                          hi = ceil(rank) (rank = fp32 q * (N - 1), at most N - 1) the bucket and the rank inside it.
 *                          q in [0, 1].  N must be < 2^32 over all ranks.
 *   aa_entropy_hist_lo   : hist (uint32[2 * 65536], zeroed here) = the low 16 bits inside lo's and hi's buckets.
 *   (across ranks the caller all-reduces hist with SUM)
 *   aa_entropy_select_lo : one block; thr[0] = lerp(v_lo, v_hi, rank - lo) as ATen forms it; NaN when N == 0 or a
 *                          counted entropy is NaN (torch.quantile's NaN). */
int aa_grpo_row_end(const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B, int32_t K,
                    int32_t *row_end, float *total, uint32_t *counter, void *stream);
int aa_entropy_hist_hi(const float *entropy, int64_t ent_stride, const int32_t *row_end, const uint8_t *mask,
                       int64_t mask_stride, int32_t B, int32_t K, uint32_t *hist, void *stream);
int aa_entropy_select_hi(const uint32_t *hist, float q, uint32_t *sel, void *stream);
int aa_entropy_hist_lo(const float *entropy, int64_t ent_stride, const int32_t *row_end, const uint8_t *mask,
                       int64_t mask_stride, int32_t B, int32_t K, const uint32_t *sel, uint32_t *hist, void *stream);
int aa_entropy_select_lo(const uint32_t *hist, const uint32_t *sel, float *thr, void *stream);

/* Clip-Cov and KL-Cov (Cui et al. 2025; verl's policy_loss.loss_mode 'clip_cov' / 'kl_cov'): the tokens whose
 * covariance cov_t = (A_t - mean A) * (lp_t - mean lp) over the counted tokens is largest lose their policy term
 * (Clip-Cov, a random share of the eligible ones) or take a |lp - old| penalty (KL-Cov, the top share).  The
 * selection runs on the device with no host sync, local to one loss call:
 *   aa_cov_moments   : one block; fixed-order fp64 (N, sum A, sum lp) over the counted tokens, each mean rounded once
 *                      to fp32 -> state.  Counted: mask[b * mask_stride + t] != 0 with advantages (B, W) of adv_dtype
 *                      and row stride adv_stride (PPO), or t < row_end[b] with fp32 per-row advantages adv[b] (GRPO);
 *                      give exactly one of mask and row_end.  log_probs (B, W) of lp_dtype.  B * W < 2^31.
 *   aa_cov_keys      : a uint32 key and a uint8 eligibility bit per flat index i = b * W + t (keys / elig, B * W
 *                      each), and hist (uint32[65536], zeroed here) = the counts of the eligible keys' high halves.
 *                      AA_COV_KL: every counted token is eligible, key = the order of fp32 cov_t (-0 = +0, NaN above
 *                      +inf).  AA_COV_CLIP: eligible = counted, not clipped (aa_ppo_actor_loss_obj's clip-fraction
 *                      predicate at [1 - clip_low, 1 + clip_high], old_log_probs NULL: ratio 1) and lb < cov_t < ub;
 *                      key = fmix32(i ^ hash_seed) (MurmurHash3's finaliser: a bijection, no ties).  mode: AA_MODE_*,
 *                      the loss kernel's rounding of the ratio.
 *   aa_cov_select_hi : one block; k = min(E, max(1, (int64)(ratio * (double)N))) of the E eligible tokens (0 when
 *                      E == 0), and the high-half bucket of the k-th largest key.  ratio = *ratio_host, a double
 *                      in (0, 1] (the product rounds as Python's int(ratio * N) does).
 *   aa_cov_hist_lo   : hist (uint32[65536], zeroed here) = the low halves of the eligible keys in that bucket.
 *   aa_cov_select_lo : one block; the threshold key T, the number of keys == T to take, and share[0] = k / N (fp32,
 *                      0 when N == 0).
 *   aa_cov_mark      : sel[b * sel_stride + t] = 1 for the k eligible tokens with the largest keys, ties at T going to
 *                      the smaller flat index; 0 elsewhere.  tie_rows: int32 [B] scratch.
 * state: uint32[16], written and read by these calls only.  Arguments are checked before any CUDA call. */
enum { AA_COV_CLIP = 1, AA_COV_KL = 2 };
int aa_cov_moments(const void *log_probs, int64_t lp_stride, int lp_dtype, const void *advantages, int64_t adv_stride,
                   int adv_dtype, const uint8_t *mask, int64_t mask_stride, const int32_t *row_end, int32_t B,
                   int32_t W, uint32_t *state, void *stream);
int aa_cov_keys(int cov_mode, const void *log_probs, int64_t lp_stride, const void *old_log_probs, int64_t old_stride,
                int lp_dtype, const void *advantages, int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                int64_t mask_stride, const int32_t *row_end, int32_t B, int32_t W, float clip_low, float clip_high,
                float lb, float ub, uint32_t hash_seed, int mode, const uint32_t *state, uint32_t *keys,
                uint8_t *elig, uint32_t *hist, void *stream);
int aa_cov_select_hi(const uint32_t *hist, const double *ratio_host, uint32_t *state, void *stream);
int aa_cov_hist_lo(const uint32_t *keys, const uint8_t *elig, int64_t n, const uint32_t *state, uint32_t *hist,
                   void *stream);
int aa_cov_select_lo(const uint32_t *hist, uint32_t *state, float *share, void *stream);
int aa_cov_mark(const uint32_t *keys, const uint8_t *elig, int32_t B, int32_t W, const uint32_t *state,
                int32_t *tie_rows, uint8_t *sel, int64_t sel_stride, void *stream);

/* aa_ppo_actor_loss_kl's objective under Clip-Cov or KL-Cov (cov_mode AA_COV_*), sel (uint8 (B, Wm), row stride
 * sel_stride) the selection of aa_cov_mark: Clip-Cov is the clip-higher objective with a selected token's term and
 * gradient 0; KL-Cov is the unclipped s = adv * ratio with s - cov_coef * |lp - old| on a selected token (cov_coef
 * finite, >= 0).  There is no dual-clip.  ref_log_probs NULL: no KL loss term (kl_loss may then be NULL).  The clip
 * fractions count the clipped branch as aa_ppo_actor_loss_obj does (0 under KL-Cov).  row_scratch: fp32 [5 * B]. */
int aa_ppo_actor_loss_cov(const void *log_probs, int64_t lp_stride, const void *old_log_probs, int64_t old_stride,
                          int lp_dtype, const void *advantages, int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                          int64_t mask_stride, int32_t B, int32_t Wm, float clip_low, float clip_high, int loss_agg,
                          int cov_mode, float cov_coef, const uint8_t *sel, int64_t sel_stride, int mode,
                          const void *ref_log_probs, int64_t ref_stride, float kl_loss_coeff, int kl_estimator,
                          float *loss, float *kl_loss, void *grad, int64_t grad_stride, float *clip_frac,
                          float *row_scratch, uint32_t *counter, void *stream);
/* aa_grpo_loss_kl's token-level objective under Clip-Cov or KL-Cov, as aa_ppo_actor_loss_cov defines them, with the
 * per-token loss -(s - beta * KL); old_log_probs NULL: ratio 1 (KL-Cov then changes nothing).  dual_clip must be 0. */
int aa_grpo_loss_cov(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                     const void *old_log_probs, int64_t old_stride, int lp_dtype, const float *advantages,
                     const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B, int32_t K,
                     float beta, float clip_low, float clip_high, int loss_agg, int kl_estimator, int cov_mode,
                     float cov_coef, const uint8_t *sel, int64_t sel_stride, int mode, float *loss, void *grad,
                     int64_t grad_stride, float *clip_frac, int32_t *row_end, float *scratch, uint32_t *counter,
                     void *stream);

/* CISPO and SAPO (TRL's GRPO loss_type 'cispo' / 'sapo'; ops.POLICY_LOSS_MODES), policy losses in place of the
 * clipped ratio, with r = exp(lp - old) rounded as aa_ppo_actor_loss_obj rounds it and s the negated loss term that
 * loss_agg aggregates:
 *   AA_PM_CISPO  w = clamp(r, max = 1 + clip_high) with its gradient stopped;  s = w * A * lp;  d s / d lp = w * A.
 *                The clip fractions count r > 1 + clip_high (the dual-clip lane is 0).
 *   AA_PM_SAPO   tau = tau_pos where A > 0, else tau_neg;  s = sigmoid(tau * (r - 1)) * 4 / tau * A (fp32: the loss
 *                and its aggregation are fp32 whatever the dtypes);  d s / d lp = 4 sigma (1 - sigma) r A.  The clip
 *                fractions are 0.
 * The modes are kept apart from AA_COV_*: the Cov entry points refuse these codes.  clip_high >= 0; tau_pos / tau_neg
 * finite and > 0 (SAPO; CISPO ignores them).  There is no dual-clip and no lower bound.  Every other argument is as in
 * aa_ppo_actor_loss_cov (ref_log_probs NULL: no KL loss term; row_scratch fp32 [5 * B]) and aa_grpo_loss_kl
 * (old_log_probs NULL: ratio 1).  Arguments are checked before any launch. */
enum { AA_PM_CISPO = 3, AA_PM_SAPO = 4 };
int aa_ppo_actor_loss_pm(const void *log_probs, int64_t lp_stride, const void *old_log_probs, int64_t old_stride,
                         int lp_dtype, const void *advantages, int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                         int64_t mask_stride, int32_t B, int32_t Wm, float clip_high, int loss_agg, int pm_mode,
                         float tau_pos, float tau_neg, int mode, const void *ref_log_probs, int64_t ref_stride,
                         float kl_loss_coeff, int kl_estimator, float *loss, float *kl_loss, void *grad,
                         int64_t grad_stride, float *clip_frac, float *row_scratch, uint32_t *counter, void *stream);
int aa_grpo_loss_pm(const void *log_probs, int64_t lp_stride, const void *ref_log_probs, int64_t ref_stride,
                    const void *old_log_probs, int64_t old_stride, int lp_dtype, const float *advantages,
                    const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t B, int32_t K,
                    float beta, float clip_high, int loss_agg, int kl_estimator, int pm_mode, float tau_pos,
                    float tau_neg, int mode, float *loss, void *grad, int64_t grad_stride, float *clip_frac,
                    int32_t *row_end, float *scratch, uint32_t *counter, void *stream);
/* K1f's actor node (aa_logprob_actor_fused_kl) and GRPO node (aa_logprob_grpo_fused_kl) under CISPO / SAPO, as
 * aa_ppo_actor_loss_pm / aa_grpo_loss_pm define them: the log-probs are bit-identical to the other K1f entry points',
 * the gradient tile carries the mode's d loss / d log-prob.  ref_log_probs (actor) NULL: no KL loss term; entropy
 * NULL: no entropy (entropy_coeff must then be 0); entropy_coeff != 0 adds the entropy bonus's gradient as the
 * _obj entry points do.  row_scratch as aa_logprob_actor_fused_kl's / aa_logprob_grpo_fused_kl's. */
int aa_logprob_actor_fused_pm(const void *logits, int logits_dtype, int64_t row_stride, int32_t V,
                              const int64_t *labels, int32_t n_segments, const int64_t *seg_logit_off,
                              const int64_t *seg_label_off, const int64_t *seg_out_off, const int64_t *seg_cum,
                              const int64_t *seg_tile_row, int64_t n_tile_rows, void *log_probs, int lp_dtype,
                              float *stat_max, float *stat_logsum, const void *old_log_probs, int64_t old_stride,
                              const void *advantages, int64_t adv_stride, int adv_dtype, const uint8_t *mask,
                              int64_t mask_stride, int32_t W, float clip_high, int loss_agg, int pm_mode,
                              float tau_pos, float tau_neg, int mode, void *grad_logits, int64_t grad_row_stride,
                              void *row_scratch, int32_t *status, float entropy_coeff, float *entropy,
                              const void *ref_log_probs, float kl_loss_coeff, int kl_estimator, void *stream);
int aa_logprob_grpo_fused_pm(const void *logits, int logits_dtype, int64_t row_stride, int32_t V, const int64_t *labels,
                             int32_t n_segments, const int64_t *seg_logit_off, const int64_t *seg_label_off,
                             const int64_t *seg_out_off, const int64_t *seg_cum, const int64_t *seg_tile_row,
                             int64_t n_tile_rows, void *log_probs, int lp_dtype, const void *ref_log_probs,
                             int64_t ref_stride, const void *old_log_probs, const float *advantages,
                             const int64_t *completion_tokens, int64_t tok_stride, int64_t eos_id, int32_t K,
                             float beta, float clip_high, int loss_agg, int kl_estimator, int pm_mode, float tau_pos,
                             float tau_neg, int mode, void *grad_logits, int64_t grad_row_stride, void *row_scratch,
                             int32_t *row_end, float *total, uint32_t *counter, int32_t *status, float *entropy,
                             float entropy_coeff, void *stream);

/* masked_mean (utils/tools.py:460-467): mean over rows of masked row means -> out[0];
 * mask == NULL: plain mean. */
int aa_masked_mean(const void *x, int dtype, int64_t x_stride, const uint8_t *mask, int64_t mask_stride,
                   int32_t B, int32_t W, float *out, float *row_scratch, uint32_t *counter, void *stream);

/* Pack the local PPO metrics (trainers/text_to_text/ppo.py:360-381) from the row statistics:
 * stats fp32 [12] = actor_loss, reward_critic_loss, reward, reward_with_kl_penalty,
 * reward_advantage, reward_return, reward_value, kl_divergence, mean_generated_length,
 * max_generated_length, status, 0 (status: the optional device status word, as in aa_dpo_loss; MAX lane).
 * Entries 0..8 are all-reduced with AVG, entries 9 and 10 with MAX; with `coll` the
 * kernel does that reduction itself over NVLink peer memory (the reference: 10 NCCL launches + a barrier). */
int aa_ppo_pack_metrics(const float *row_stats, const float *reward, const float *value_row_mean,
                        const float *actor_loss, const float *critic_loss, int32_t B, float *stats,
                        const aa_coll *coll, const int32_t *status, void *stream);

/* The same one-shot NVLink all-reduce on its own: dst[0..n) = reduce over ranks of src[0..n), n <= 16 floats, src may
 * equal dst.  The DPO trainer launches it on a side stream right after K2, so that the wait for the slowest rank
 * overlaps K1b instead of sitting between K2 and K1b on the critical path. */
int aa_allreduce_packed(const float *src, float *dst, int32_t n, const aa_coll *coll, void *stream);

/* ---------------------------------------------------------------------------------------
 * K6  lm_head x log-prob in one kernel (SURVEY.md 8f rank 1; rows that carry no gradient):
 *   out[r] = log_softmax(hidden[r, :] @ weight^T)[labels[r]]
 * = gather_log_probabilities(lm_head(hidden), labels) (utils/tools.py:402-413 on the output of the model's
 * nn.Linear lm_head; callers trainers/text_to_text/dpo.py:128 (reference model), ppo.py:266-267 (rollout))
 * without the (n_rows, V) logits tile.  hidden (n_rows, H) and weight (V, H) are bf16, K-major, rows
 * 16-byte aligned (strides in elements, multiples of 8), H a multiple of 64; V is arbitrary (128257 works:
 * the odd leading dimension only exists in the tile that is never written).  wgmma (m64n256k16 per warpgroup,
 * fp32 accumulators in registers), operands staged by TMA into a 4-stage 128-byte-swizzled ring, epilogue =
 * online (max, sum-exp) + label pick on the accumulator registers.  FAITHFUL: each logit is rounded to bf16 before
 * the softmax (the rounding point of nn.Linear) and the result is rounded to bf16.  stat_max / stat_logsum
 * (optional, n_rows fp32 each) receive the row statistics.  `partial` (optional, `partial_floats` fp32 of
 * device scratch; 3 * 132 * 128 always suffices on a 132-SM H100): with fewer 128-row tiles than SMs the vocabulary is also
 * split across CTAs and the per-split (max, sum, label logit) are merged by a second tiny launch.  Needs a driver that exports
 * cuTensorMapEncodeTiled (resolved at run time; the library does not link libcuda).
 * Work: 2 * n_rows * H * V flops; HBM: weight + hidden read ~once (the weight sweep stays in L2).
 * ------------------------------------------------------------------------------------- */
int aa_linear_logprob_fwd(const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride,
                          const void *weight, int32_t V, int64_t weight_row_stride, const int64_t *labels,
                          void *out, int out_dtype, float *stat_max, float *stat_logsum, float *partial,
                          int64_t partial_floats, int mode, int32_t *status, void *stream);

/* K6 with the entropy of every row: entropy fp32 [n_rows], H = -sum_j p_j log p_j over the logits the statistics fold
 * (bf16-rounded in FAITHFUL mode, the fp32 accumulators in F32 mode), never rounded.  The (max, sum-exp, entropy sum)
 * merge across the quad and across vocabulary splits uses t' = alpha (t + (m - m') s); `partial` then holds FOUR floats
 * per (row, split): 4 * 132 * 128 always suffices on a 132-SM H100 (with fewer floats the split count is lowered as for
 * K6).  out, stat_max and stat_logsum are bit-identical to aa_linear_logprob_fwd's when both launches split the
 * vocabulary the same way: `partial` NULL, or partial_floats >= 4 * n_rows * splits for the split count `splits` that
 * aa_linear_logprob_fwd picks.  A buffer sized at 3 floats per split for the plain launch can make this launch split
 * fewer ways; the statistics are then merged in another order and may differ in the last bits. */
int aa_linear_logprob_fwd_entropy(const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride,
                                  const void *weight, int32_t V, int64_t weight_row_stride, const int64_t *labels,
                                  void *out, int out_dtype, float *stat_max, float *stat_logsum, float *partial,
                                  int64_t partial_floats, int mode, int32_t *status, float *entropy, void *stream);

/* K6s: K6 with a second epilogue on the same accumulator tile -- every logit is rounded to bf16 (nn.Linear's rounding
 * point, in both modes: the stored tile is bf16) and stored into `logits` (n_rows, ld), ld >= ceil(V / 256) * 256 and a
 * multiple of 8 (columns >= V are written as +0), while (max, sum-exp, label logit) are folded from the same rounded
 * values.  Everything else is aa_linear_logprob_fwd: `out` (FAITHFUL: the log-prob rounded to bf16; F32: not rounded),
 * stat_max / stat_logsum, `partial` and the split-vocabulary merge, NaN and AA_STATUS_LABEL_OOB on an out-of-range
 * label.  The forward of a loss whose gradient seed is known before any logit exists (the mean cross-entropy: every
 * valid row's upstream gradient is -loss_scale / n_valid) then runs K1b on the stored tile instead of recomputing it
 * in the backward (K6b): three GEMM passes over 2 * n_rows * H * V instead of four. */
int aa_linear_logits(const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride,
                     const void *weight, int32_t V, int64_t weight_row_stride, const int64_t *labels,
                     void *out, int out_dtype, float *stat_max, float *stat_logsum, float *partial,
                     int64_t partial_floats, int mode, int32_t *status, void *logits, int64_t ld, void *stream);

/* K6b: K6's pipeline with a store epilogue -- the first of the three backward kernels of the fused lm_head x
 * log-prob path.  Recomputes the logits tile on the tensor cores and writes
 *   dlogits[r, j] = g[r] * ([j == labels[r]] - softmax_j)      (bf16; FAITHFUL: softmax from the rounded log-softmax)
 * into a (n_rows, ld) buffer, ld >= ceil(V / 256) * 256 and a multiple of 8 (columns >= V are written as 0), from the
 * (max, logsum) K6 saved -- the "recompute + K1b" step of the lm_head backward in one kernel; d(hidden) and d(weight)
 * are aa_linear_dhidden / aa_linear_dweight on that buffer. */
int aa_linear_dlogits(const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride,
                      const void *weight, int32_t V, int64_t weight_row_stride, const int64_t *labels,
                      const float *stat_max, const float *stat_logsum, const void *grad_rows,
                      int grad_rows_dtype, void *dlogits, int64_t ld, int mode, void *stream);
/* aa_linear_dlogits with the gradient of each row's entropy added in the epilogue (entropy bonus):
 *   d(logits)[row, k] += -g_H * p_k * (l_k + H)   with the p_k and l_k of the line above, in fp32 before the bf16 store,
 * 0 for a -inf logit.  entropy: the fp32 H of aa_linear_logprob_fwd_entropy; grad_entropy: g_H per row
 * (grad_entropy_dtype).  Rows with g_H == 0 are bit-identical to aa_linear_dlogits's. */
int aa_linear_dlogits_entropy(const void *hidden, int64_t n_rows, int32_t H, int64_t hidden_row_stride,
                              const void *weight, int32_t V, int64_t weight_row_stride, const int64_t *labels,
                              const float *stat_max, const float *stat_logsum, const void *grad_rows,
                              int grad_rows_dtype, const float *entropy, const void *grad_entropy,
                              int grad_entropy_dtype, void *dlogits, int64_t ld, int mode, void *stream);

/* The two GEMMs that finish that backward: the autograd of the model's nn.Linear lm_head (callers
 * trainers/text_to_text/dpo.py:128, ppo.py:338) given the d(logits) buffer of aa_linear_dlogits.  Same wgmma / TMA
 * pipeline as K6 (128 x 256 tiles, fp32 accumulation), persistent grid, operands read in place:
 *   aa_linear_dhidden:  d_hidden (n_rows, H) bf16 = dlogits (n_rows, ld) . weight (V, H)       [columns >= V of dlogits
 *                       must be zero; the weight is consumed MN-major, vocabulary rows >= V are zero-filled by TMA]
 *   aa_linear_dweight:  (V, H) result = [acc_f32 if accumulate] + dlogits^T . hidden (n_rows, H), both operands MN-major.
 *                       Written to acc_f32 (fp32, row stride acc_row_stride) when d_weight == NULL, else rounded to bf16
 *                       into d_weight.  Row chunks: first chunk accumulate = 0, d_weight = NULL; middle chunks
 *                       accumulate = 1, d_weight = NULL; last chunk accumulate = 1, d_weight given -- one rounding at the
 *                       end, like a single GEMM over all rows.  A single chunk needs no fp32 buffer at all.
 * ld: multiple of 64, >= V; H: multiple of 64; all bases 16-byte aligned. */
int aa_linear_dhidden(const void *dlogits, int64_t n_rows, int64_t ld, const void *weight, int32_t V, int32_t H,
                      int64_t weight_row_stride, void *d_hidden, int64_t d_hidden_row_stride, void *stream);
int aa_linear_dweight(const void *dlogits, int64_t n_rows, int64_t ld, const void *hidden, int32_t H,
                      int64_t hidden_row_stride, int32_t V, float *acc_f32, int64_t acc_row_stride, int32_t accumulate,
                      void *d_weight, int64_t d_weight_row_stride, void *stream);

/* ---------------------------------------------------------------------------------------
 * Integer layout kernels (bit-exact).
 * move_padding_left : trainers/text_image_to_text/ppo.py:56-87 (utils/tools.py:615-639)
 * count_nonpad      : the host `.tolist()` bookkeeping at text_image_to_text/ppo.py:190-203
 *                     (response_len = nonpad(sequence) - nonpad(prompt))
 * ------------------------------------------------------------------------------------- */
int aa_move_padding_left(const int64_t *ids, int32_t B, int32_t L, int64_t row_stride, int64_t pad_id,
                         int64_t *out, void *stream);
int aa_count_nonpad(const int64_t *ids, int32_t B, int32_t L, int64_t row_stride, int64_t pad_id,
                    int32_t *counts, void *stream);

/* Everything trainers/text_image_to_text/ppo.py:185-203 does after `generate`, in one launch and without the host:
 * moved = move_padding_left(sequences) (B, L) int64; attention_mask = moved != pad (B, L) bytes (torch.bool);
 * response_lens[b] = max(nonpad(sequences[b]) - nonpad(prompt_ids[b]), 0) int32 (the reference: two `.tolist()` and a
 * Python list filter per sample). */
int aa_ppo_rollout_layout(const int64_t *prompt_ids, int32_t P, int64_t prompt_row_stride, const int64_t *sequences,
                          int32_t L, int64_t seq_row_stride, int32_t B, int64_t pad_id, int64_t *moved,
                          uint8_t *attention_mask, int32_t *response_lens, void *stream);

/* The K1 / K1b row plan of per-sample response tails built from DEVICE response lengths (the reference slices each
 * sample on the host, text_image_to_text/ppo.py:229-239).  table: int64 [5][B + 1] = seg_logit_off, seg_label_off,
 * seg_out_off, seg_cum, seg_tile_row as aa_logprob_fwd / aa_logprob_bwd take them (pass n_rows = B * width, the kernels
 * read the exact total from seg_cum[B]; the backward runs in tile mode, n_tile_rows = B * seq).  Sample b scores
 * n_b = clamp(lens[b] - label_shift, 0, width) rows from tile position seq - lens[b] + row_shift on, against
 * labels[b * label_row_stride + (label_tail_len > 0 ? label_tail_len - lens[b] : 0) + label_shift + j], results at
 * out[b * width + j].  Lengths that do not fit set AA_STATUS_SHORT_SEQUENCE and are clamped.
 * copies > 1 (table: [5][copies * B + 1]): the plan repeated for `copies` identically shaped logits tensors lying
 * copy_logit_delta ELEMENTS apart (their base pointers differ by that much), results copy_out_delta apart -- the actor
 * and the reference model of a rollout are then scored by ONE aa_logprob_fwd launch (forward only). */
int aa_tail_plan_build(const int32_t *response_lens, int32_t B, int32_t seq, int64_t sample_stride, int64_t row_stride,
                       int64_t label_row_stride, int32_t label_tail_len, int32_t label_shift, int32_t row_shift,
                       int32_t width, int32_t copies, int64_t copy_logit_delta, int64_t copy_out_delta, int64_t *table,
                       int32_t *status, void *stream);

/* pad_sequence([x[b][-R_b:] for b], batch_first=True) -- trainers/text_image_to_text/ppo.py:233-249 (rollout) and
 * :318-330 (rl_step: critic values), a Python loop + pad_sequence in the reference -- and its adjoint.
 * One tail rule, the one the critic's tail load and aa_tail_plan_build use: R_b = clamp(lens[b], 0, W), and the tail is
 * columns [W - R_b, W - R_b + n_b) of the width-W row, n_b = min(R_b, Rmax).
 *   adjoint = 0:  src (B, W), out (B, Rmax):  out[b, k] = k < n_b ? src[b, W - R_b + k] : 0
 *   adjoint = 1:  src (B, Rmax), out (B, W):  out[b, j] = W - R_b <= j < W - R_b + n_b ? src[b, j - (W - R_b)] : 0
 *                 (the gradient: the exact transpose of adjoint = 0)
 * src / out hold `dtype` elements (bit copies); lens (B,) int32 on the device, Rmax <= W.  Lengths in [0, Rmax] are the
 * intended use; any other int32 length follows the rule above, and no access leaves row b of src or out. */
int aa_tail_rows(const void *src, int dtype, int64_t src_row_stride, const int32_t *lens, int32_t B, int32_t W,
                 int32_t Rmax, void *out, int64_t out_row_stride, int32_t adjoint, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* AA_B200_H_ */
