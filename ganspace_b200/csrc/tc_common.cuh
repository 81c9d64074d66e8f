// wgmma / TMA / mbarrier PTX wrappers shared by the tensor-core kernels (gram_tc.cu, mapping_tc.cu), the fp32 -> fp16 hi/lo
// operand split, and the declarations of the tensor-core entry points that other files call.  sm_90a (Hopper).  The
// shared-memory descriptor encoding follows cute::GMMA::GmmaDescriptor.
//
// Warp layout: warpgroups 0 and 1 (warps 0-7) are the MMA consumers and keep their accumulators in registers; warp 8 holds
// the TMA producer (one elected thread).  In the Gram kernel (gram_tc.cu: the batch statistics of stats_tc.cu and the
// large-d small side of bigd.cu) each consumer warpgroup owns 64 rows of a 128-row tile; mapping_tc.cu gives each whole
// 128 x 128 tiles in turns and makes warps 8-11 a producer warpgroup (setmaxnreg).
#pragma once
#include "common.cuh"
#include <cuda.h>
#include <cuda_fp16.h>

namespace gsb {
namespace tc {

constexpr int CONSUMER_THREADS = 256;                // two warpgroups
constexpr int THREADS = CONSUMER_THREADS + 32;       // + the producer warp
constexpr int PRODUCER_WARP = CONSUMER_THREADS / 32;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "TCW_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, 0x989680;\n\t"
        "@P1 bra TCW_DONE;\n\t"
        "bra TCW_LOOP;\n\t"
        "TCW_DONE:\n\t"
        "}" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

// ---- TMA --------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap *map, uint64_t *bar, void *dst, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap *map, uint64_t *bar, void *dst, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap *map, const void *src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}

// ---- wgmma ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// all but the most recently committed wgmma group have completed
__device__ __forceinline__ void wgmma_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// K-major, SWIZZLE_128B shared-memory matrix descriptor (tile base 1024-byte aligned):
//   [0,14) start>>4 | [16,30) LBO>>4 (unused for swizzled K-major) | [32,46) SBO>>4 (8 rows * 128 B = 1024)
//   [62,64) layout = 1 (SWIZZLE_128B).  One K step of 16 fp16 = +32 B = +2 on the start field.
__device__ __forceinline__ uint64_t sw128_kmajor_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// D[64 x 128] (+)= A[64 x 16] B[128 x 16]^T, fp16 operands from shared memory, fp32 accumulator in registers.
// Fragment of thread t (warp w = t/32 of the warpgroup, lane l): d[i] is row 16 w + l/4 + 8 ((i >> 1) & 1),
// column 8 (i >> 2) + 2 (l % 4) + (i & 1).
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate)
        : "memory");
}

// one K-block of 64 of the three-MMA split product  D (+)= A_hi B_hi + A_lo B_hi + A_hi B_lo  on a 64 x 128 accumulator
__device__ __forceinline__ void split_kblock_m64n128(float (&d)[64], uint64_t ah, uint64_t al, uint64_t bh, uint64_t bl,
                                                     bool accumulate) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint64_t koff = (uint64_t)(2 * k);          // +32 B per K step of 16
        wgmma_m64n128(d, ah + koff, bh + koff, (accumulate || k > 0) ? 1u : 0u);
        wgmma_m64n128(d, al + koff, bh + koff, 1u);
        wgmma_m64n128(d, ah + koff, bl + koff, 1u);
    }
}

// ---- fp32 -> fp16 hi/lo split (22 significant bits): x = hi + lo, hi = fp16(x), lo = fp16(x - hi) -----------------------
__device__ __forceinline__ void split1(float x, __half &hi, __half &lo) {
    hi = __float2half_rn(x);
    lo = __float2half_rn(x - __half2float(hi));
}
// two values, packed as half2 bit patterns (a in the low half)
__device__ __forceinline__ void split2(float a, float b, uint32_t &hi, uint32_t &lo) {
    __half h0, h1, l0, l1;
    split1(a, h0, l0);
    split1(b, h1, l1);
    hi = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
    lo = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
}
// four values, packed as 4 x fp16 (8 bytes); returns whether any |f| exceeds 60000 (hi would be at or near fp16's range end)
__device__ __forceinline__ bool split4(const float (&f)[4], uint2 &hi, uint2 &lo) {
    split2(f[0], f[1], hi.x, lo.x);
    split2(f[2], f[3], hi.y, lo.y);
    return (fabsf(f[0]) > 60000.f) | (fabsf(f[1]) > 60000.f) | (fabsf(f[2]) > 60000.f) | (fabsf(f[3]) > 60000.f);
}
// split4 stored at hi + off and lo + off (off a multiple of 4); ovf |= the overflow test
__device__ __forceinline__ void store_split4(const float (&f)[4], __half *hi, __half *lo, int64_t off, bool &ovf) {
    uint2 ph, pl;
    ovf |= split4(f, ph, pl);
    *reinterpret_cast<uint2 *>(hi + off) = ph;
    *reinterpret_cast<uint2 *>(lo + off) = pl;
}

}  // namespace tc

// ---- host: tensor maps (core.cu) -------------------------------------------------------------------------------------
// fp16 or fp32 tensor, innermost dimension contiguous, 128B swizzle, L2 promotion 256 B, out-of-bounds elements read as zero;
// dims / box innermost first; strides (bytes) of dims 1..rank-1
int tc_make_tmap(CUtensorMap *map, CUtensorMapDataType type, const void *base, int rank, const uint64_t *dims,
                 const uint64_t *strides_bytes, const uint32_t *box);

// ---- entry points used across files ----------------------------------------------------------------------------------
// Gram kernel with promoted accumulation (gram_tc.cu).  Operands: n_groups fp16 hi/lo matrices of n_pad rows x k columns,
// rows k_pitch elements apart, scaled by powers of two 2^e.
//   Store:      out[g] = 2^-2e_g (x x^T)_g for each group (exps: [n_groups]; n_rows == n_pad, a multiple of 128); every
//               entry is written, so out need not be zeroed
//   Accumulate: out += 2^-(e_i + e_j) (x x^T)_ij for i, j < n_rows of the one group (exps: [n_pad], one per row); out is
//               summed into with fp64 atomics over 4096-column chunks of k
enum class GramEpilogue { Store, Accumulate };
int gram_tc_launch(GramEpilogue epi, const __half *hi, const __half *lo, int64_t k, int64_t k_pitch, int n_groups, int n_pad,
                   int n_rows, const int *exps, double *out, cudaStream_t st);
// Store Grams of up to GRAM_GROUPED_MAX operand sets of different widths in one launch (gram_tc.cu): for each set, out[g] as
// gram_tc_launch(Store, hi, lo, nb, nbp, n_groups, d, d, exps, out) computes it, with the same bits; work items are
// (set, group, tile pair), set-major
constexpr int GRAM_GROUPED_MAX = 32;
struct GramGroupedOperand {
    const __half *hi, *lo;      // [n_groups][d][nbp]
    int64_t nb, nbp;
    int d, n_groups;            // d % 128 == 0
    const int *exps;            // [n_groups]
    double *out;                // [n_groups][d][d]
};
int gram_tc_grouped_launch(const GramGroupedOperand *ops, int n, cudaStream_t st);
// large-d small side T = M M^T (gram_tc.cu)
size_t gram_tc_workspace_bytes(int n_pad, int64_t d);
bool gram_tc_supported(int64_t d);
int gram_tc(const float *M, int n_rows, int n_pad, int64_t d, void *ws, double *T, cudaStream_t st);

// batch means and centred Grams of consecutive row groups (stats_tc.cu)
bool stats_tc_supported(int64_t nb, int d);
size_t stats_tc_workspace_bytes(int n_groups, int64_t nb, int d);
int stats_tc(const float *x, int n_groups, int64_t nb, int d, int64_t ld, double *mean, double *gram, void *ws, cudaStream_t st);
// the same for several inputs (gsb_batch_stats_grouped; widths d % 128 == 0, d <= 1024), each with stats_tc's bits
bool stats_tc_grouped_width(int d);
size_t stats_tc_grouped_workspace_bytes(const gsb_stats_desc *descs, int n_desc);
int stats_tc_grouped(const gsb_stats_desc *descs, int n_desc, void *ws, cudaStream_t st);

// mapping network, dense layers and the conv tap GEMM on the persistent layer kernel (mapping_tc.cu)
size_t mapping_tc_packed_bytes(int n_layers, int dim);
int mapping_tc_pack(const float *pw, int n_layers, int dim, void *tc_base, cudaStream_t st);
int mapping_forward_tc(const float *pb, void *tc_base, int n_layers, int dim, const float *d_z, float *d_w,
                       int64_t n, bool pixelnorm, void *ws, int leave_free_sms, cudaStream_t st);
size_t mapping_tc_workspace_bytes(int64_t n, int dim);
unsigned *mapping_tc_overflow_flag(void *tc_base, int n_layers, int dim);
size_t tc_linear_workspace_bytes(int64_t n, int N, int K);
int tc_linear(const float *x, const float *w, const float *bias, float *y, int64_t n, int N, int K, bool lrelu, void *ws,
              cudaStream_t st);
int tc_gemm_plain(const __half *a_hi, const __half *a_lo, int64_t M, int K, const __half *w_hi, const __half *w_lo, int N,
                  const float *inv_wscale, float *out, unsigned *overflow, unsigned *queue, int leave_free_sms, cudaStream_t st);
// The weight operand of tc_gemm_plain and of the mapping layers from fp32 W [rows, cols, taps] (taps fastest).  The operand is
// w' = scale W 2^s, with the power of two that puts max |w'| in [8192, 16384): hi keeps its 11 bits and lo = fp16(w' - hi) stays
// a normal fp16 number.  Writes
//   scal [3]          {inv_wscale = 2^-s (the pointer the GEMM takes), wscale = 2^s, absmax = max |scale W|}; scal[2] must be
//                     zero on entry (it is an atomic max)
//   hi, lo [n_pad, cols]  row tap' rows + r = w'[r, :, tap], tap' = tap or, with reverse_taps, taps - 1 - tap; rows from
//                     taps rows to n_pad (a multiple of 32, the GEMM's N) are zero
//   wsq [rows, cols]  (unless nullptr) the sum over taps, in tap order, of (scale W)^2 as an fmaf chain
// Stream-ordered, no host sync.
int tc_split_weight(const float *w, int rows, int cols, int taps, float scale, bool reverse_taps, int n_pad, __half *hi, __half *lo,
                    float *scal, float *wsq, cudaStream_t st);

}  // namespace gsb
