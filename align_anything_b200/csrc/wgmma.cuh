// wgmma.cuh -- the sm_90a tensor-core plumbing shared by the lm_head kernels (K6 / K6b in linear_logprob.cu, the two
// backward GEMMs in linear_backward.cu): mbarriers, TMA tile loads, wgmma.mma_async and its shared-memory descriptors.
//
// Every kernel built on it has the same shape: one producer thread streams 128 x 64 tiles of A and 256 x 64 tiles of B
// (bf16, 128-byte swizzle) into a STAGES-deep shared-memory ring with cp.async.bulk.tensor, and two consumer
// warpgroups each multiply their 64 rows of A by the whole B tile with wgmma m64n256k16 into 128 fp32 registers per
// thread; a third warpgroup hosts the producer.  The descriptors follow the canonical GMMA layouts documented in
// CUTLASS (cute/arch/mma_sm90_desc.hpp, `make_gmma_desc` in cute/atom/mma_traits_sm90_gmma.hpp).
#pragma once

#include <cuda.h>

#include "common.cuh"

namespace aa {
namespace wg {

constexpr int BM = 128, BN = 256, BK = 64, WG_K = 16;
constexpr int A_BYTES = BM * BK * 2, B_BYTES = BN * BK * 2, STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int STAGES = 4;                           // 4 x 48 KB of the 227 KB a block may reserve
constexpr int CONSUMER_THREADS = 256;               // warpgroups 0 and 1: rows [0, 64) and [64, 128) of the tile
constexpr int THREADS = CONSUMER_THREADS + 128;     // warpgroup 2: TMA producer (one thread issues)
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /* alignment slack */ + 256 /* barriers */;
constexpr int ACC = BN / 2;                         // fp32 accumulators per consumer thread (m64n256)

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
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
      "WG_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WG_DONE;\n"
      "bra WG_WAIT;\n"
      "WG_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int c_inner, int c_outer, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c_inner), "r"(c_outer), "r"(smem_u32(bar))
      : "memory");
}

// ---- shared-memory matrix descriptors (SWIZZLE_128B: layout type 1 in bits 62-63) -----------------------------------
// K-major operand tile as TMA writes it with the 128-byte swizzle and a {64 (K), rows} box: rows of 128 bytes (64 bf16
// along K), 8-row atoms of 1024 bytes.  start address >> 4 | LBO = 1 (unused: one swizzle atom along K) | SBO = 1024 B
// between 8-row atoms.  One wgmma consumes K = 16 = 32 bytes of every row: the k-th slice of a 64-wide block starts
// 32 * k bytes into the (swizzled) row.
__device__ __forceinline__ uint64_t desc_k_major(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3ffffu) >> 4);
  d |= 1ull << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= 1ull << 62;
  return d;
}
// MN-major operand tile (the M / N index is the contiguous one in global memory): TMA box {64 (MN), BK (K rows)} with
// the 128-byte swizzle gives, per 64-wide MN chunk, BK rows of 128 bytes = BK / 8 atoms of (64 MN x 8 K) -- the
// canonical layout  Swizzle<3,4,3> o ((8,n),(8,k)):((1,LBO),(8,SBO))  in 16-byte units: 8 K rows 128 B apart inside an
// atom, SBO = 1024 B from one group of 8 K rows to the next, LBO = distance between consecutive 64-wide MN chunks
// (each chunk is loaded by its own TMA box: LBO = BK * 128 B).  One wgmma consumes K = 16 rows = 2 atoms = 2048 bytes.
__device__ __forceinline__ uint64_t desc_mn_major(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3ffffu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3fffu) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= 1ull << 62;
  return d;
}
// k-th 16-deep slice of an operand tile; `tile_addr` already points at the consumer's 64-row half for A
template <int MN_MAJOR>
__device__ __forceinline__ uint64_t operand_desc(uint32_t tile_addr, int k_slice) {
  if (MN_MAJOR) return desc_mn_major(tile_addr + static_cast<uint32_t>(k_slice) * (WG_K * 128), BK * 128);
  return desc_k_major(tile_addr + static_cast<uint32_t>(k_slice) * (WG_K * 2));
}
// byte offset of consumer warpgroup `w`'s 64 rows inside an A tile: 64 K-major rows of 128 B, or the w-th 64-wide
// MN chunk -- both 8 KB
__device__ __forceinline__ uint32_t a_half_offset(int w) { return static_cast<uint32_t>(w) * (64 * 128); }

// Register split between the warpgroups (the block is launched with 65536 / 384 = 168 per thread): the producer gives
// registers back, the consumers take them for the 128 accumulators plus the epilogue.  40 + 2 * 232 <= 3 * 168.
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory"); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// D (64 x 256, fp32, registers) (+)= A (64 x 16, smem) . B (256 x 16, smem)^T; bf16 operands, A_MN / B_MN = 1 for an
// MN-major operand (the transpose bits of the instruction)
template <int A_MN, int B_MN>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[ACC], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79,"
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111,"
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, %131, %132;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(accumulate), "n"(A_MN), "n"(B_MN));
}
// Accumulator fragment of m64nN (PTX ISA, "wgmma register fragment D"): thread t of the warpgroup holds, for i in
// [0, N / 2), the element (row, col) = (16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2), 8 * (i / 4) + 2 * (t % 4) + i % 2).
__device__ __forceinline__ int frag_row(int t, int i) { return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int t, int i) { return 8 * (i >> 2) + 2 * (t & 3) + (i & 1); }

// Consumer side of one output tile: acc = A (this warpgroup's 64 rows) . B^T over `k_blocks` ring stages.  `it` counts
// ring stages across tiles (stage = it % STAGES, parity = (it / STAGES) & 1).  A stage is released (all 256 consumer
// threads arrive on empty[s]) once the wgmmas that read it have completed: one k-block stays in flight behind the one
// being issued.
template <int A_MN, int B_MN>
__device__ __forceinline__ void consume_tile(float (&acc)[ACC], uint8_t *tiles, uint64_t *full, uint64_t *empty,
                                             int k_blocks, int64_t &it, int w) {
  int prev = -1;
  for (int kb = 0; kb < k_blocks; ++kb, ++it) {
    const int s = static_cast<int>(it % STAGES);
    mbar_wait(full + s, static_cast<uint32_t>((it / STAGES) & 1));
    const uint32_t a = smem_u32(tiles + s * STAGE_BYTES) + a_half_offset(w), b = smem_u32(tiles + s * STAGE_BYTES) + A_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / WG_K; ++k)
      wgmma_m64n256k16<A_MN, B_MN>(acc, operand_desc<A_MN>(a, k), operand_desc<B_MN>(b, k), (kb | k) != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0) mbar_arrive(empty + prev);
    prev = s;
  }
  wgmma_wait<0>();
  mbar_arrive(empty + prev);
}

// ---- host: TMA tensor maps (cuTensorMapEncodeTiled resolved through the runtime: no libcuda link) ------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void *sym = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(sym);
  }
  return fn;
}
// 2-D bf16 tensor: `inner` contiguous elements per row, `rows` rows `row_stride` elements apart; box = 64 inner
// elements (one 128-byte swizzle span) x box_rows; elements outside the tensor read as zero.
inline int make_map_2d(CUtensorMap *map, const void *base, int64_t inner, int64_t rows, int64_t row_stride, int box_rows,
                       const char *who) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    set_error("%s: cuTensorMapEncodeTiled is not available from the driver", who);
    return AA_ERR_UNSUPPORTED;
  }
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(row_stride) * 2};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(BK), static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t elem[2] = {1, 1};
  auto encode = [&] {
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), dims, strides, box, elem,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  };
  CUresult r = encode();
  if (r == CUDA_ERROR_INVALID_CONTEXT) {
    // The driver call needs a current context, and a thread whose first CUDA work is this launch has none yet (the
    // autograd engine's device thread when the lm_head backward is the first node it runs).  cudaSetDevice binds the
    // device's primary context to the thread, as the runtime's own first launch would.
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaSetDevice(dev) == cudaSuccess) r = encode();
  }
  if (r != CUDA_SUCCESS) {
    set_error("%s: cuTensorMapEncodeTiled failed (%d)", who, static_cast<int>(r));
    return AA_ERR_ARG;
  }
  return AA_OK;
}

}  // namespace wg
}  // namespace aa
