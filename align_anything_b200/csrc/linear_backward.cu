// linear_backward.cu -- the two GEMMs that finish the backward of the fused lm_head x log-prob path (SURVEY.md 8f rank 1):
//
//   d(hidden) (n, H)  = dlogits (n, V) . weight (V, H)              aa_linear_dhidden
//   d(weight) (V, H) += dlogits^T (V, n) . hidden (n, H)            aa_linear_dweight
//
// i.e. the autograd of the model's `nn.Linear` lm_head (callers trainers/text_to_text/dpo.py:128, ppo.py:338) given the
// d(logits) tile that K6b (linear_logprob.cu) recomputes on the tensor cores.  Both run on the K6 pipeline (wgmma.cuh) --
// a producer thread streams TMA boxes into a 4-stage 128-byte-swizzled ring, two consumer warpgroups multiply with
// wgmma m64n256k16 into fp32 registers and write their 64 x 256 slice of the tile -- as ONE persistent kernel template
// whose operands may be K-major or MN-major:
//
//   d(hidden): A = dlogits, K-major (K = vocabulary, contiguous);  B = weight seen as (N = H, K = V): H is the contiguous
//              index of `weight`, so B is MN-major -- no transposed or padded copy of the 1 GB weight is ever made;
//              vocabulary rows >= V are zero-filled by TMA.
//   d(weight): A = dlogits seen as (M = V, K = n) and B = hidden seen as (N = H, K = n): both MN-major.
//
// MN-major tiles are brought in as 64-wide boxes (one swizzle span) of BK rows each; the shared-memory descriptors
// (wgmma.cuh) describe that layout directly, the transpose bits of the instruction select it.
// Persistent grid: CTA b walks tiles b, b + grid, ... with the N tiles of one M tile adjacent, so the CTAs resident
// together share their A strip through L2.  d(weight) accumulates across row chunks in an fp32 buffer (read-modify-write
// in the epilogue) and is rounded to bf16 once, by the last chunk -- like a single GEMM over all rows.
#include <atomic>

#include "wgmma.cuh"

namespace aa {
namespace lmbwd {

using namespace wg;

struct GemmParams {
  int M, N, K;               // C (M x N) = A (M x K) . B (N x K)^T
  __nv_bfloat16 *c_bf16;     // optional (M, N) bf16 result, row stride ldc_bf16
  int64_t ldc_bf16;
  float *c_f32;              // optional (M, N) fp32 accumulator, row stride ldc_f32
  int64_t ldc_f32;
  int beta;                  // != 0: add the fp32 accumulator's current contents
  int tiles_m, tiles_n;
};

// linear tile id -> (M tile, N tile).  The N tiles of one M tile are adjacent, so co-resident CTAs share the A strip.
__device__ __forceinline__ void tile_coords(const GemmParams &p, int tile, int &mt, int &nt) {
  mt = tile / p.tiles_n;
  nt = tile % p.tiles_n;
}

template <int A_MN, int B_MN>
__global__ void __launch_bounds__(THREADS, 1)
    lm_head_bwd_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                            const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t *full = reinterpret_cast<uint64_t *>(tiles + STAGES * STAGE_BYTES);
  uint64_t *empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_tiles = p.tiles_m * p.tiles_n;
  const int k_blocks = (p.K + BK - 1) / BK;

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
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int mt, nt;
        tile_coords(p, tile, mt, nt);
        const int m0 = mt * BM, n0 = nt * BN;
        for (int kb = 0; kb < k_blocks; ++kb, ++it) {
          const int s = static_cast<int>(it % STAGES);
          mbar_wait(empty + s, static_cast<uint32_t>((it / STAGES) & 1) ^ 1u);
          uint8_t *a = tiles + s * STAGE_BYTES, *b = a + A_BYTES;
          mbar_expect_tx(full + s, STAGE_BYTES);
          if (A_MN) {  // inner coordinate = M, outer = K rows; one box per 64-wide M chunk
#pragma unroll
            for (int c = 0; c < BM / 64; ++c) tma_load_2d(a + c * (BK * 128), &map_a, m0 + 64 * c, kb * BK, full + s);
          } else {
            tma_load_2d(a, &map_a, kb * BK, m0, full + s);
          }
          if (B_MN) {
#pragma unroll
            for (int c = 0; c < BN / 64; ++c) tma_load_2d(b + c * (BK * 128), &map_b, n0 + 64 * c, kb * BK, full + s);
          } else {
            tma_load_2d(b, &map_b, kb * BK, n0, full + s);
          }
        }
      }
    }
    return;
  }

  // ------------------------------- consumers: wgmma + epilogue ----------------------------
  consumer_regs();
  const int w = threadIdx.x >> 7, t = threadIdx.x & 127;
  float acc[ACC];
  int64_t it = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int mt, nt;
    tile_coords(p, tile, mt, nt);
    const int m0 = mt * BM + 64 * w, n0 = nt * BN;
    consume_tile<A_MN, B_MN>(acc, tiles, full, empty, k_blocks, it, w);
#pragma unroll
    for (int i = 0; i < ACC; i += 2) {  // (i, i + 1): one row, two adjacent columns
      const int64_t row = m0 + frag_row(t, i);
      const int col = n0 + frag_col(t, i);
      if (row >= p.M || col >= p.N) continue;  // N is a multiple of 64: a pair never straddles it
      float v0 = acc[i], v1 = acc[i + 1];
      if (p.beta) {
        const float2 o = *reinterpret_cast<const float2 *>(p.c_f32 + row * p.ldc_f32 + col);
        v0 += o.x;
        v1 += o.y;
      }
      if (p.c_bf16)
        *reinterpret_cast<uint32_t *>(p.c_bf16 + row * p.ldc_bf16 + col) = pack2<__nv_bfloat16>(v0, v1);
      else
        *reinterpret_cast<float2 *>(p.c_f32 + row * p.ldc_f32 + col) = make_float2(v0, v1);
    }
  }
}

template <int A_MN, int B_MN>
static int launch(const CUtensorMap &map_a, const CUtensorMap &map_b, const GemmParams &p, cudaStream_t st, const char *who) {
  auto kern = lm_head_bwd_gemm_kernel<A_MN, B_MN>;
  static std::atomic<bool> configured{false};  // the attribute is idempotent: a race sets it twice, harmlessly
  if (!configured.load(std::memory_order_relaxed)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) {
      set_error("%s: %s", who, cudaGetErrorString(e));
      return static_cast<int>(e);
    }
    configured.store(true, std::memory_order_relaxed);
  }
  const int total = p.tiles_m * p.tiles_n;
  const int grid = total < sm_count() ? total : sm_count();
  kern<<<grid, THREADS, SMEM_BYTES, st>>>(map_a, map_b, p);
  return check_launch(who);
}

static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace lmbwd
}  // namespace aa

using namespace aa;

extern "C" int aa_linear_dhidden(const void *dlogits, int64_t n_rows, int64_t ld, const void *weight, int32_t V, int32_t H,
                                 int64_t weight_row_stride, void *d_hidden, int64_t d_hidden_row_stride, void *stream) {
  AA_REQUIRE(n_rows >= 0 && V > 0 && H > 0, AA_ERR_ARG, "aa_linear_dhidden: bad sizes");
  if (n_rows == 0) return AA_OK;
  AA_REQUIRE(dlogits && weight && d_hidden, AA_ERR_ARG, "aa_linear_dhidden: null pointer");
  AA_REQUIRE(H % 64 == 0, AA_ERR_UNSUPPORTED, "aa_linear_dhidden: H=%d must be a multiple of 64", H);
  AA_REQUIRE(ld >= V && ld % 64 == 0, AA_ERR_ALIGN, "aa_linear_dhidden: ld must be >= V and a multiple of 64");
  AA_REQUIRE(lmbwd::aligned16(dlogits) && lmbwd::aligned16(weight) && lmbwd::aligned16(d_hidden) &&
                 weight_row_stride % 8 == 0 && weight_row_stride >= H && d_hidden_row_stride % 8 == 0 &&
                 d_hidden_row_stride >= H,
             AA_ERR_ALIGN, "aa_linear_dhidden: operands must be 16-byte aligned with 16-byte row strides");
  AA_REQUIRE(n_rows < (int64_t(1) << 31) - wg::BM, AA_ERR_UNSUPPORTED, "aa_linear_dhidden: too many rows");
  CUtensorMap map_a, map_b;
  // A = dlogits (n_rows, ld): K-major, box 64 (K) x 128 rows.  Columns [V, ld) are zero (K6b writes them so).
  int rc = wg::make_map_2d(&map_a, dlogits, ld, n_rows, ld, wg::BM, "aa_linear_dhidden");
  if (rc) return rc;
  // B = weight (V, H) read as (N = H contiguous, K = V rows): MN-major, box 64 (N) x 64 (K rows); rows >= V read as zero
  rc = wg::make_map_2d(&map_b, weight, H, V, weight_row_stride, wg::BK, "aa_linear_dhidden");
  if (rc) return rc;
  lmbwd::GemmParams p{static_cast<int>(n_rows), H, static_cast<int>(ld), static_cast<__nv_bfloat16 *>(d_hidden),
                      d_hidden_row_stride, nullptr, 0, 0, static_cast<int>((n_rows + wg::BM - 1) / wg::BM),
                      (H + wg::BN - 1) / wg::BN};
  return lmbwd::launch<0, 1>(map_a, map_b, p, static_cast<cudaStream_t>(stream), "aa_linear_dhidden");
}

extern "C" int aa_linear_dweight(const void *dlogits, int64_t n_rows, int64_t ld, const void *hidden, int32_t H,
                                 int64_t hidden_row_stride, int32_t V, float *acc_f32, int64_t acc_row_stride,
                                 int32_t accumulate, void *d_weight, int64_t d_weight_row_stride, void *stream) {
  AA_REQUIRE(n_rows > 0 && V > 0 && H > 0, AA_ERR_ARG, "aa_linear_dweight: bad sizes (an empty row chunk has no GEMM)");
  AA_REQUIRE(acc_f32 || d_weight, AA_ERR_ARG, "aa_linear_dweight: no output given");
  AA_REQUIRE(!accumulate || acc_f32, AA_ERR_ARG, "aa_linear_dweight: accumulate needs the fp32 accumulator");
  AA_REQUIRE(dlogits && hidden, AA_ERR_ARG, "aa_linear_dweight: null pointer");
  AA_REQUIRE(H % 64 == 0, AA_ERR_UNSUPPORTED, "aa_linear_dweight: H=%d must be a multiple of 64", H);
  AA_REQUIRE(ld >= V && ld % 64 == 0, AA_ERR_ALIGN, "aa_linear_dweight: ld must be >= V and a multiple of 64");
  AA_REQUIRE(lmbwd::aligned16(dlogits) && lmbwd::aligned16(hidden) && lmbwd::aligned16(acc_f32) && lmbwd::aligned16(d_weight) &&
                 hidden_row_stride % 8 == 0 && hidden_row_stride >= H &&
                 (!acc_f32 || (acc_row_stride % 4 == 0 && acc_row_stride >= H)) &&
                 (!d_weight || (d_weight_row_stride % 8 == 0 && d_weight_row_stride >= H)),
             AA_ERR_ALIGN, "aa_linear_dweight: operands must be 16-byte aligned with 16-byte row strides");
  AA_REQUIRE(n_rows < (int64_t(1) << 31) - wg::BK, AA_ERR_UNSUPPORTED, "aa_linear_dweight: too many rows");
  CUtensorMap map_a, map_b;
  // A = dlogits (n_rows, ld) read as (M = vocabulary contiguous, K = rows): MN-major
  int rc = wg::make_map_2d(&map_a, dlogits, ld, n_rows, ld, wg::BK, "aa_linear_dweight");
  if (rc) return rc;
  // B = hidden (n_rows, H) read as (N = H contiguous, K = rows): MN-major
  rc = wg::make_map_2d(&map_b, hidden, H, n_rows, hidden_row_stride, wg::BK, "aa_linear_dweight");
  if (rc) return rc;
  lmbwd::GemmParams p{V, H, static_cast<int>(n_rows), static_cast<__nv_bfloat16 *>(d_weight), d_weight_row_stride, acc_f32,
                      acc_row_stride, accumulate ? 1 : 0, (V + wg::BM - 1) / wg::BM, (H + wg::BN - 1) / wg::BN};
  return lmbwd::launch<1, 1>(map_a, map_b, p, static_cast<cudaStream_t>(stream), "aa_linear_dweight");
}
