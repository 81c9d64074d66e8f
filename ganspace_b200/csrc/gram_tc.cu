// Gram matrices on the Hopper tensor cores (wgmma + TMA) with a PROMOTED accumulator: the centred per-group Grams of the
// batch statistics (stats_tc.cu) and the small-side Gram  T = M M^T  of the large-d IPCA engine.
//
// Part of the replacement of sklearn IncrementalPCA.partial_fit (_incremental_pca.py:254-380) for conv feature maps
// (bigd.cu): M is sklearn's stacked matrix [S*Vt; X - mean_b; correction] ([n_s <= 4096, d ~ 5e5] fp32 in HBM).
//
// Precision.  As in mapping_tc.cu every fp32 operand is split x 2^e = hi + lo into two fp16 numbers (22 significant
// bits; e = a power-of-two exponent per row of M, or per group of centred samples, chosen so that hi keeps 11 bits and
// lo stays a normal fp16), and a product is three MMAs (hi hi, lo hi, hi lo) accumulated in fp32.  Tensor-core accumulation
// TRUNCATES when aligning addends, which is harmless over K = 512 but not over K = 524288.  So the MMAs accumulate only
// FLUSH_KB * 64 = 256 values of K (48 MMA steps) into the wgmma accumulator; that partial is then added into a second set
// of fp32 REGISTERS with round-to-nearest.  At the end of a work item the sums are scaled back by the exact power of two
// and written in fp64, mirrored across the diagonal:
//     Store       (batch statistics) one work item covers a whole group: plain stores of each group's Gram
//     Accumulate  (large-d) one work item covers a chunk of 4096 columns: RED.ADD.F64 into T.  Error budget per entry:
//                 <= 48 x 2^-24 truncation inside a flush, round-to-nearest fp32 across the 16 flushes of a chunk, fp64
//                 across chunks.
//
// Kernel: persistent, one CTA per SM, 128 x 128 x 64 tiles (upper tile pairs only), 3 smem stages x 64 KB (A_hi, A_lo,
// B_hi, B_lo; both operands are row blocks of the same two fp16 matrices; diagonal tiles load B too: reading B from A's slot
// instead made the kernel 3 % slower for the large-d Gram and 10 % slower for the d = 512 statistics on an H100 80GB HBM3 at
// 700 W), SWIZZLE_128B K-major, 3-D TMA boxes {64 columns of K, 128 rows, 1 group}; columns past K are zero-filled by the
// TMA unit:
//     warp 8     TMA producer
//     warps 0-7  two warpgroups of 64 output rows each: wgmma m64n128k16, promotion, epilogue
// Work items are (group, chunk of K, tile pair) with the tile pair fastest and then the chunk: group-major for the
// statistics, chunk-major for the large-d Gram, so the CTAs running at the same time read the same 2112 x 4096 slab of M
// (35 MB as hi+lo) out of the 50 MB L2.
#include "tc_common.cuh"
#include <math.h>
#include <string.h>

namespace gsb {
namespace gtc {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int STAGES = 3;
constexpr int FLUSH_KB = 4;                 // K-blocks (of 64) accumulated by the MMAs before the promotion into registers
constexpr int CHUNK_KB = 64;                // K-blocks per work item of the Accumulate epilogue (4096 columns of d)
constexpr uint32_t TILE_BYTES = BM * BK * 2;               // 16 KB
constexpr uint32_t STAGE_BYTES = 4 * TILE_BYTES;           // 64 KB
constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;

struct Params {
    double *out;            // Store: [n_groups][ld][ld];  Accumulate: [ld][ld], summed into
    const int *exps;        // scale exponents of the split operands: Store: [n_groups];  Accumulate: [ld], one per row
    int ld, n_rows;         // output leading dimension; rows (and columns) of the Gram
    int nt, npairs;         // upper tile pairs of the nt x nt grid of 128-row blocks
    int n_groups, n_chunks;
    int total_kb, chunk_kb; // K-blocks per group, per work item
};

// gram_tc_grouped_launch: up to GRAM_GROUPED_MAX operand sets of different widths in one persistent grid (Store epilogue)
struct GroupedGramDesc {
    double *out;            // [n_groups][d][d]
    const int *exps;        // [n_groups]
    int d, nt, npairs, total_kb;
    int item0;              // first work item of the descriptor
};
struct GroupedGramParams {
    CUtensorMap tm[GRAM_GROUPED_MAX][2];      // hi, lo operand maps of each descriptor
    GroupedGramDesc desc[GRAM_GROUPED_MAX];
    int n_desc, num_items;
};

struct Item { int g, m0, n0, kb0, kb1; };

// work item -> (group, chunk of K, tile pair), tile pair fastest
__device__ __forceinline__ Item decode_tile(int item, int nt, int npairs, int n_chunks, int chunk_kb, int total_kb) {
    const int outer = item / npairs;
    int pair = item % npairs, ti = 0;
    while (pair >= nt - ti) { pair -= nt - ti; ++ti; }
    Item w;
    w.g = outer / n_chunks;
    w.kb0 = (outer % n_chunks) * chunk_kb;
    w.kb1 = (w.kb0 + chunk_kb < total_kb) ? w.kb0 + chunk_kb : total_kb;
    w.m0 = ti * BM;
    w.n0 = (ti + pair) * BN;
    return w;
}

// What a work item reads and writes: its operand maps and its output Gram(s)
struct Target {
    const CUtensorMap *hi, *lo;
    double *out;
    const int *exps;
    int ld, n_rows;
};

// the work items of one gram_tc_launch: one pair of operand maps, one output
struct PlainItems {
    const CUtensorMap *hi, *lo;
    const Params *p;
    __device__ __forceinline__ int count() const { return p->n_groups * p->n_chunks * p->npairs; }
    __device__ __forceinline__ void prefetch(int lane) const { if (lane == 0) { tc::tma_prefetch_desc(hi); tc::tma_prefetch_desc(lo); } }
    __device__ __forceinline__ Item decode(int item, Target &t) const {
        t.hi = hi; t.lo = lo; t.out = p->out; t.exps = p->exps; t.ld = p->ld; t.n_rows = p->n_rows;
        return decode_tile(item, p->nt, p->npairs, p->n_chunks, p->chunk_kb, p->total_kb);
    }
};

// the work items of gram_tc_grouped_launch: (descriptor, group, tile pair), descriptor-major, each descriptor with its own maps,
// width and Store output
struct GroupedItems {
    const GroupedGramParams *p;
    __device__ __forceinline__ int count() const { return p->num_items; }
    __device__ __forceinline__ void prefetch(int lane) const {
        if (lane < p->n_desc) { tc::tma_prefetch_desc(&p->tm[lane][0]); tc::tma_prefetch_desc(&p->tm[lane][1]); }
    }
    __device__ __forceinline__ Item decode(int item, Target &t) const {
        int i = 0;
        while (i + 1 < p->n_desc && item >= p->desc[i + 1].item0) ++i;
        const GroupedGramDesc &g = p->desc[i];
        t.hi = &p->tm[i][0]; t.lo = &p->tm[i][1]; t.out = g.out; t.exps = g.exps; t.ld = g.d; t.n_rows = g.d;
        return decode_tile(item - g.item0, g.nt, g.npairs, 1, g.total_kb, g.total_kb);
    }
};

// The persistent kernel body, shared by both work-item maps: the producer and the MMA / promotion / epilogue code are the same
// instructions whichever map decodes the items, so a Gram computed through either map has the same bits.
template <GramEpilogue EPI, class Items>
__device__ __forceinline__ void gram_tc_body(const Items &items) {
    using namespace tc;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + STAGES * STAGE_BYTES);
    uint64_t *full_bar = bars;                     // [STAGES]
    uint64_t *empty_bar = bars + STAGES;           // [STAGES]: one arrival per consumer warp

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_items = items.count();

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CONSUMER_THREADS / 32); }
        mbar_fence_init();
    }
    if (warp == PRODUCER_WARP) items.prefetch(lane);
    __syncthreads();

    if (warp == PRODUCER_WARP) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            int stage = 0; uint32_t phase = 0;
            for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
                Target t;
                const Item w = items.decode(item, t);
                for (int kb = w.kb0; kb < w.kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t *st = smem + stage * STAGE_BYTES;
                    mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
                    tma_load_3d(t.hi, &full_bar[stage], st, kb * BK, w.m0, w.g);
                    tma_load_3d(t.lo, &full_bar[stage], st + TILE_BYTES, kb * BK, w.m0, w.g);
                    tma_load_3d(t.hi, &full_bar[stage], st + 2 * TILE_BYTES, kb * BK, w.n0, w.g);
                    tma_load_3d(t.lo, &full_bar[stage], st + 3 * TILE_BYTES, kb * BK, w.n0, w.g);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== MMA + promoted accumulation + epilogue =====================
        const int wg = warp >> 2;                       // 64-row half of the 128-row tile
        const int row_frag = wg * 64 + (warp & 3) * 16 + (lane >> 2), col_frag = 2 * (lane & 3);
        int stage = 0; uint32_t phase = 0;
        float acc[64], r[64];
#pragma unroll
        for (int j = 0; j < 64; ++j) { acc[j] = 0.f; r[j] = 0.f; }
        for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
            Target t;
            const Item w = items.decode(item, t);
            const int nkb = w.kb1 - w.kb0;
            for (int g0 = 0; g0 < nkb; g0 += FLUSH_KB) {
                const int g1 = (g0 + FLUSH_KB < nkb) ? g0 + FLUSH_KB : nkb;
                for (int kb = g0; kb < g1; ++kb) {
                    mbar_wait(&full_bar[stage], phase);
                    const uint32_t st = smem_u32(smem + stage * STAGE_BYTES);
                    const uint32_t sa = st + (uint32_t)wg * (TILE_BYTES / 2);
                    wgmma_fence();
                    split_kblock_m64n128(acc, sw128_kmajor_desc(sa), sw128_kmajor_desc(sa + TILE_BYTES),
                                         sw128_kmajor_desc(st + 2 * TILE_BYTES), sw128_kmajor_desc(st + 3 * TILE_BYTES), kb > g0);
                    wgmma_commit();
                    wgmma_wait_all();
                    if (lane == 0) mbar_arrive(&empty_bar[stage]);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
#pragma unroll
                for (int j = 0; j < 64; ++j) r[j] = __fadd_rn(r[j], acc[j]);
            }
            if constexpr (EPI == GramEpilogue::Store) {
                const double unscale = ldexp(1.0, -2 * __ldg(t.exps + w.g));
                double *G = t.out + (size_t)w.g * t.ld * t.ld;
                const bool diag = (w.m0 == w.n0);
#pragma unroll
                for (int j = 0; j < 64; j += 2) {
                    const int gm = w.m0 + row_frag + 8 * ((j >> 1) & 1), gn = w.n0 + 8 * (j >> 2) + col_frag;
                    const double v0 = (double)r[j] * unscale, v1 = (double)r[j + 1] * unscale;
                    if (!diag) {
                        *reinterpret_cast<double2 *>(G + (size_t)gm * t.ld + gn) = make_double2(v0, v1);
                        G[(size_t)gn * t.ld + gm] = v0;
                        G[(size_t)(gn + 1) * t.ld + gm] = v1;
                    } else {
                        // diagonal tile: (i,j) and (j,i) come out of differently ordered MMA sums; keep the upper triangle
                        // and mirror it, so the chain reads an exactly symmetric matrix
                        if (gn >= gm) { G[(size_t)gm * t.ld + gn] = v0; G[(size_t)gn * t.ld + gm] = v0; }
                        if (gn + 1 >= gm) { G[(size_t)gm * t.ld + gn + 1] = v1; G[(size_t)(gn + 1) * t.ld + gm] = v1; }
                    }
                }
            } else {
                const int gm0 = w.m0 + row_frag, gm1 = gm0 + 8;
                const int em0 = gm0 < t.n_rows ? __ldg(&t.exps[gm0]) : 0, em1 = gm1 < t.n_rows ? __ldg(&t.exps[gm1]) : 0;
#pragma unroll
                for (int j = 0; j < 64; ++j) {
                    const int gm = ((j >> 1) & 1) ? gm1 : gm0, gn = w.n0 + 8 * (j >> 2) + col_frag + (j & 1);
                    if (gm < t.n_rows && gn < t.n_rows && gn >= gm) {
                        // 2^-(e_i + e_j) as an fp64 bit pattern: exact, |e_i + e_j| stays far inside the normal range
                        const int e = ((j >> 1) & 1 ? em1 : em0) + __ldg(&t.exps[gn]);
                        const double val = (double)r[j] * __hiloint2double((1023 - e) << 20, 0);
                        atomicAdd(&t.out[(size_t)gm * t.ld + gn], val);
                        if (gn > gm) atomicAdd(&t.out[(size_t)gn * t.ld + gm], val);
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < 64; ++j) r[j] = 0.f;
        }
    }
}

template <GramEpilogue EPI>
__global__ void __launch_bounds__(tc::THREADS, 1)
gram_tc_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo, const __grid_constant__ Params p) {
    gram_tc_body<EPI>(PlainItems{&tm_hi, &tm_lo, &p});
}

__global__ void __launch_bounds__(tc::THREADS, 1)
gram_tc_grouped_kernel(const __grid_constant__ GroupedGramParams p) {
    gram_tc_body<GramEpilogue::Store>(GroupedItems{&p});
}

// ---- operand preparation ----------------------------------------------------------------------------------
// per-row exponent e: the row maximum times 2^e lies in [8192, 16384) (hi keeps 11 bits, lo stays a normal fp16)
__global__ void __launch_bounds__(1024)
row_exponent_kernel(const float *__restrict__ M, int64_t d, int n_rows, int *__restrict__ rexp) {
    __shared__ float red[32];
    const int r = blockIdx.x, tid = threadIdx.x;
    float m = 0.f;
    if (r < n_rows) {
        const float4 *row = reinterpret_cast<const float4 *>(M + (size_t)r * d);
        for (int64_t i = tid; i < d / 4; i += 1024) {
            const float4 v = row[i];
            m = fmaxf(fmaxf(m, fabsf(v.x)), fmaxf(fabsf(v.y), fmaxf(fabsf(v.z), fabsf(v.w))));
        }
    }
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) red[tid >> 5] = m;
    __syncthreads();
    if (tid < 32) {
        m = red[tid];
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (tid == 0) {
            int e = 0;
            if (m > 0.f && m < 3.0e38f) { int ex; frexpf(m, &ex); e = 14 - ex; }
            rexp[r] = e;
        }
    }
}
// columns [k0, k0 + w) of every row of M (row pitch ld) -> fp16 hi / lo rows of pitch w
__global__ void __launch_bounds__(256)
row_split_kernel(const float *__restrict__ M, int64_t ld, int64_t k0, int64_t w, int n_rows, const int *__restrict__ rexp,
                 __half *__restrict__ hi, __half *__restrict__ lo) {
    const int r = blockIdx.y;
    const int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;           // float4 index within the slab of the row
    if (q >= w / 4) return;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < n_rows) v = reinterpret_cast<const float4 *>(M + (size_t)r * ld + k0)[q];
    const float sc = ldexpf(1.f, rexp[r]);
    const float f[4] = {v.x * sc, v.y * sc, v.z * sc, v.w * sc};              // power-of-two scale: exact
    uint2 ph, pl;
    tc::split4(f, ph, pl);
    reinterpret_cast<uint2 *>(hi + (size_t)r * w)[q] = ph;
    reinterpret_cast<uint2 *>(lo + (size_t)r * w)[q] = pl;
}

}  // namespace gtc

int gram_tc_launch(GramEpilogue epi, const __half *hi, const __half *lo, int64_t k, int64_t k_pitch, int n_groups, int n_pad,
                   int n_rows, const int *exps, double *out, cudaStream_t st) {
    using namespace gtc;
    if (int r = raise_dyn_smem(gram_tc_kernel<GramEpilogue::Store>, SMEM_BYTES)) return r;
    if (int r = raise_dyn_smem(gram_tc_kernel<GramEpilogue::Accumulate>, SMEM_BYTES)) return r;
    CUtensorMap tm_hi, tm_lo;
    const uint64_t dims[3] = {(uint64_t)k, (uint64_t)n_pad, (uint64_t)n_groups};
    const uint64_t strides[2] = {(uint64_t)k_pitch * 2, (uint64_t)n_pad * k_pitch * 2};
    const uint32_t box[3] = {(uint32_t)BK, (uint32_t)BM, 1};
    if (int r = tc_make_tmap(&tm_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, hi, 3, dims, strides, box)) return r;
    if (int r = tc_make_tmap(&tm_lo, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, lo, 3, dims, strides, box)) return r;
    Params p;
    p.out = out; p.exps = exps; p.ld = n_pad; p.n_rows = n_rows;
    p.nt = (n_rows + BM - 1) / BM;
    p.npairs = p.nt * (p.nt + 1) / 2;
    p.n_groups = n_groups;
    p.total_kb = (int)((k + BK - 1) / BK);
    // a stored Gram has to be complete in one work item; an accumulated one is split into chunks of K that share the L2
    p.chunk_kb = (epi == GramEpilogue::Store) ? p.total_kb : CHUNK_KB;
    p.n_chunks = (p.total_kb + p.chunk_kb - 1) / p.chunk_kb;
    const int items = p.n_groups * p.n_chunks * p.npairs;
    const int grid = items < num_sms() ? items : num_sms();
    if (epi == GramEpilogue::Store)
        gram_tc_kernel<GramEpilogue::Store><<<grid, tc::THREADS, SMEM_BYTES, st>>>(tm_hi, tm_lo, p);
    else
        gram_tc_kernel<GramEpilogue::Accumulate><<<grid, tc::THREADS, SMEM_BYTES, st>>>(tm_hi, tm_lo, p);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// Store Grams of several operand sets (stats_tc_grouped): work items (descriptor, group, tile pair) flattened into one grid
int gram_tc_grouped_launch(const GramGroupedOperand *ops, int n, cudaStream_t st) {
    using namespace gtc;
    GSB_CHECK_ARG(n > 0 && n <= GRAM_GROUPED_MAX, "gram_tc_grouped_launch: 0 < n <= %d descriptors (n=%d)", GRAM_GROUPED_MAX, n);
    if (int r = raise_dyn_smem(gram_tc_grouped_kernel, SMEM_BYTES)) return r;
    GroupedGramParams p;
    memset(&p, 0, sizeof(p));
    int items = 0;
    for (int i = 0; i < n; ++i) {
        const GramGroupedOperand &o = ops[i];
        const uint64_t dims[3] = {(uint64_t)o.nb, (uint64_t)o.d, (uint64_t)o.n_groups};
        const uint64_t strides[2] = {(uint64_t)o.nbp * 2, (uint64_t)o.d * o.nbp * 2};
        const uint32_t box[3] = {(uint32_t)BK, (uint32_t)BM, 1};
        if (int r = tc_make_tmap(&p.tm[i][0], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, o.hi, 3, dims, strides, box)) return r;
        if (int r = tc_make_tmap(&p.tm[i][1], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, o.lo, 3, dims, strides, box)) return r;
        GroupedGramDesc &g = p.desc[i];
        g.out = o.out; g.exps = o.exps; g.d = o.d;
        g.nt = (o.d + BM - 1) / BM;
        g.npairs = g.nt * (g.nt + 1) / 2;
        g.total_kb = (int)((o.nb + BK - 1) / BK);
        g.item0 = items;
        items += o.n_groups * g.npairs;
    }
    p.n_desc = n;
    p.num_items = items;
    const int grid = items < num_sms() ? items : num_sms();
    gram_tc_grouped_kernel<<<grid, tc::THREADS, SMEM_BYTES, st>>>(p);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// The fp16 operands cover at most GRAM_TC_SLAB columns of d at a time: wider rows (StyleGAN2 convs.6 .. convs.9, d = 2 M / 4 M)
// are converted and multiplied slab by slab into the same T, so the operand copy stays 4.4 GB at n_pad = 2112 instead of
// growing with d (35 GB at d = 4,194,304).  Widths up to one slab (config 5's d = 524,288) run as one launch, as before.
constexpr int64_t GRAM_TC_SLAB = 524288;
static int64_t gram_tc_slab(int64_t d) { return d < GRAM_TC_SLAB ? d : GRAM_TC_SLAB; }

size_t gram_tc_workspace_bytes(int n_pad, int64_t d) {
    return 2 * align_up((size_t)n_pad * gram_tc_slab(d) * 2, 256) + align_up((size_t)n_pad * sizeof(int), 256);
}
bool gram_tc_supported(int64_t d) { return d % 64 == 0; }

// T[n_pad, n_pad] (fp64, zeroed by the caller) += M[0:n_rows] M[0:n_rows]^T.  ws: gram_tc_workspace_bytes(n_pad, d).
// The per-row exponents come from the whole row, so every slab is split with the same scale and the slabs' partial sums add up
// exactly as the chunks of one launch do (fp64 atomics into T).
int gram_tc(const float *M, int n_rows, int n_pad, int64_t d, void *ws, double *T, cudaStream_t st) {
    using namespace gtc;
    GSB_CHECK_ARG(gram_tc_supported(d) && n_rows <= n_pad, "gram_tc: d %% 64 != 0");
    const int64_t slab = gram_tc_slab(d);
    const size_t hb = align_up((size_t)n_pad * slab * 2, 256);
    __half *hi = reinterpret_cast<__half *>(ws);
    __half *lo = reinterpret_cast<__half *>(reinterpret_cast<char *>(ws) + hb);
    int *rexp = reinterpret_cast<int *>(reinterpret_cast<char *>(ws) + 2 * hb);
    row_exponent_kernel<<<n_pad, 1024, 0, st>>>(M, d, n_rows, rexp);
    GSB_CHECK_LAUNCH();
    for (int64_t k0 = 0; k0 < d; k0 += slab) {
        const int64_t w = (d - k0 < slab) ? d - k0 : slab;                      // a multiple of 64, as d and slab are
        dim3 sg((unsigned)((w / 4 + 255) / 256), (unsigned)n_pad);
        row_split_kernel<<<sg, 256, 0, st>>>(M, d, k0, w, n_rows, rexp, hi, lo);
        GSB_CHECK_LAUNCH();
        if (int r = gram_tc_launch(GramEpilogue::Accumulate, hi, lo, w, w, 1, n_pad, n_rows, rexp, T, st)) return r;
    }
    return GSB_OK;
}

}  // namespace gsb
