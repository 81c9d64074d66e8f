// StyleGAN2 mapping network on the Hopper tensor cores (wgmma + TMA), fp32-grade accuracy.
//
// Replaces models/stylegan2/stylegan2-pytorch/model.py:151-161 (EqualLinear.forward: F.linear(x, W*scale)
// then fused bias + leaky-ReLU(0.2)*sqrt2, op/fused_act.py:86-92) for the 8 layers of Generator.style.
//
// Precision.  The parity target (principal directions vs sklearn on the same seeds, cos >= 0.999 at relative
// eigen-gaps of 0.27 %) needs ~1e-6 relative accuracy per layer: single-pass bf16/fp16 (2^-9 / 2^-12) fails
// it (SURVEY.md section 7 hard part 3).  Each fp32 operand is split into two fp16 numbers, x = hi + lo with
// hi = fp16(x), lo = fp16(x - hi)  (22 significant bits), and the product is formed from three MMAs
//     D += A_hi W_hi ;  D += A_lo W_hi ;  D += A_hi W_lo          (fp32 accumulation)
// dropping only the lo*lo term (2^-24).  Weights are pre-scaled by a per-layer power of two so that W_lo
// stays in fp16's normal range; the scale is undone exactly in the epilogue.  fp16 (11-bit significand) at
// the bf16 MMA rate gives this accuracy in 3 MMAs; TF32 would need 3 MMAs at half the rate.
//
// Kernel (one launch per layer; activations travel between layers as fp16 hi/lo pairs = the same 4 B/element
// as fp32): persistent, one CTA per SM, warp-specialised, ping-pong: each consumer warpgroup owns whole 128 x 128 output
// tiles, and the two take turns on the tensor cores, so that one's epilogue runs under the other's MMAs:
//     warps 8-11  producer warpgroup: one thread claims the CTA's tiles from the launch's queue and issues their TMA loads in
//                 order (A_hi, A_lo, W_hi, W_lo: 128 x 64 boxes; SWIZZLE_128B, K-major); the warpgroup hands most of its
//                 registers to the consumers (setmaxnreg)
//     warps 0-7   two consumer warpgroups; tile i of the CTA belongs to warpgroup i & 1.  Main loop: wgmma m64n128k16 on
//                 rows 0-63 and 64-127 of the tile, 6 per K step of 16 each (the accumulator, 128 fp32 per thread, lives in
//                 registers), one wgmma group kept in flight.  A warpgroup starts its main loop when the other has issued
//                 all of its own (an mbarrier hand-over per tile), then runs the epilogue (2^-s, +bias, leaky-ReLU, *sqrt2
//                 -> split to fp16 hi/lo for the next layer, or fp32 for the last layer) through a swizzled shared-memory
//                 staging box and TMA stores while the other warpgroup's MMAs run
// smem: 3 stages x 64 KB (A_hi, A_lo, W_hi, W_lo: 16 KB each) with mbarrier full/empty pairs, + 2 x 16 KB staging, + one
// tile slot per consumer warpgroup with its own full/empty mbarrier pair.
// Tiles are claimed in order (n fastest) with an atomicAdd on a per-launch counter, one at a time as the producer issues the
// last k-block of its current tile.  The launch shares the GPU with other streams (the RNG's launch groups take SMs as a
// layer launch drains), and a CTA that starts late simply takes fewer tiles, where a static split (CTA b: tiles b, b + grid,
// ...) would make the whole layer wait for its share.  Results do not depend on which CTA computes a tile.
#include "tc_common.cuh"
#include <stdlib.h>

namespace gsb {

constexpr int TC_BLOCK_M = 128;
constexpr int TC_BLOCK_N = 128;
constexpr int TC_BLOCK_K = 64;           // 64 fp16 = one 128-byte swizzle row
constexpr int TC_STAGES = 3;
constexpr int TC_FRAG_ROWS = 64;         // rows of one m64n128 accumulator fragment (two per tile)
constexpr uint32_t TC_A_BYTES = TC_BLOCK_M * TC_BLOCK_K * 2;   // 16 KB
constexpr uint32_t TC_W_BYTES = TC_BLOCK_N * TC_BLOCK_K * 2;   // 16 KB
constexpr uint32_t TC_STAGE_BYTES = 2 * TC_A_BYTES + 2 * TC_W_BYTES;   // 64 KB
constexpr uint32_t TC_BOX_BYTES = TC_FRAG_ROWS * 128;           // one 64-row x 128-byte output box: 8 KB
constexpr uint32_t TC_STAGING_BYTES = 2 * 2 * TC_BOX_BYTES;     // per warpgroup: (hi, lo) of 64 columns, or 2 x 32 fp32 columns
// a whole producer warpgroup, so that setmaxnreg can move registers to the consumers: 40 + 2 x 232 per thread of each
// sub-partition's three warps fits its 16K registers (with 9 warps and no redistribution the cap is 168 and the 128-float
// accumulator spills)
constexpr int TC_THREADS = tc::CONSUMER_THREADS + 128;
constexpr uint32_t TC_SMEM_BYTES = TC_STAGES * TC_STAGE_BYTES + TC_STAGING_BYTES + 128 /*barriers, tile slots*/ + 1024 /*align slack*/;
static_assert(TC_SMEM_BYTES <= 232448, "mapping_layer_tc_kernel: shared memory exceeds the H100's 227 KB per block");

struct TcParams {
    const float *bias;      // [N_total] pre-multiplied by lr_mul
    __half *out_hi;         // next layer's A_hi [M, N_total] (nullptr on the last layer)
    __half *out_lo;
    float *out_f32;         // fp32 output [M, N_total] (last layer)
    unsigned *overflow;     // set to 1 when an activation leaves fp16's range
    unsigned *queue;        // tile claim counter, zeroed before the launch
    const float *inv_wscale;   // device pointer to 2^-s of this layer
    int M, N_total, K;
    int mode;               // 0: (acc 2^-s + bias) -> leaky-ReLU * sqrt2 (EqualLinear);  1: plain acc 2^-s (tc_gemm_plain);  2: acc 2^-s + bias
    int dbg;                // profiling experiments (GANSPACE_B200_MAPPING_DBG): 1 no stores, 2 no W loads, 4 no A loads, 8 no MMAs
};

__global__ void __launch_bounds__(TC_THREADS, 1)
mapping_layer_tc_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                        const __grid_constant__ CUtensorMap tm_w_hi, const __grid_constant__ CUtensorMap tm_w_lo,
                        const __grid_constant__ CUtensorMap tm_o0, const __grid_constant__ CUtensorMap tm_o1,
                        const TcParams p) {
    using namespace tc;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t *staging = smem + TC_STAGES * TC_STAGE_BYTES;
    uint64_t *bars = reinterpret_cast<uint64_t *>(staging + TC_STAGING_BYTES);
    uint64_t *full_bar = bars;                         // [TC_STAGES]
    uint64_t *empty_bar = bars + TC_STAGES;            // [TC_STAGES]: one arrival per warp of the consuming warpgroup
    uint64_t *turn_bar = bars + 2 * TC_STAGES;         // [2]: warpgroup wg may start its next main loop (arrivals: the other's warps)
    uint64_t *tile_full = bars + 2 * TC_STAGES + 2;    // [2]: tile_slot[wg] holds warpgroup wg's next tile (arrival: the producer)
    uint64_t *tile_empty = bars + 2 * TC_STAGES + 4;   // [2]: warpgroup wg has read tile_slot[wg] (arrivals: its warps)
    volatile int *tile_slot = reinterpret_cast<volatile int *>(bars + 2 * TC_STAGES + 6);   // [2]: tile number, -1 = no more

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int num_m_tiles = (p.M + TC_BLOCK_M - 1) / TC_BLOCK_M;
    // N and K need not be multiples of the tile: the TMA unit zero-fills operand rows / columns past the tensor's extent and
    // clips stores (the 128/64/32-channel StyledConv blocks: N = 9 cout = 1152 / 576 / 288, K = cin down to 32)
    const int num_n_tiles = (p.N_total + TC_BLOCK_N - 1) / TC_BLOCK_N;
    const int num_k_blocks = (p.K + TC_BLOCK_K - 1) / TC_BLOCK_K;
    // work unit = one 128 x 128 output tile, N fastest: neighbouring claims read the same A rows while they are in L2.  The
    // CTA's i-th claimed unit belongs to consumer warpgroup i & 1.
    const int num_units = num_m_tiles * num_n_tiles;

    if (threadIdx.x == 0) {
        for (int s = 0; s < TC_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
        for (int w = 0; w < 2; ++w) { mbar_init(&turn_bar[w], 4); mbar_init(&tile_full[w], 1); mbar_init(&tile_empty[w], 4); }
        mbar_fence_init();
    }
    if (warp == PRODUCER_WARP && lane == 0) {
        tma_prefetch_desc(&tm_a_hi); tma_prefetch_desc(&tm_a_lo);
        tma_prefetch_desc(&tm_w_hi); tma_prefetch_desc(&tm_w_lo);
        tma_prefetch_desc(&tm_o0); tma_prefetch_desc(&tm_o1);
    }
    __syncthreads();

    if (warp >= PRODUCER_WARP) {
        // ===================== TMA producer =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == PRODUCER_WARP && lane == 0) {
            int stage = 0; uint32_t phase = 0;
            int u = (int)atomicAdd(p.queue, 1u);
            for (int i = 0;; ++i) {
                const int wg = i & 1;
                mbar_wait(&tile_empty[wg], ((uint32_t)(i >> 1) & 1) ^ 1);   // warpgroup wg has taken its previous tile
                if (u >= num_units) {                                      // no more tiles: tell both warpgroups
                    tile_slot[wg] = -1;
                    mbar_arrive(&tile_full[wg]);
                    mbar_wait(&tile_empty[wg ^ 1], ((uint32_t)((i + 1) >> 1) & 1) ^ 1);
                    tile_slot[wg ^ 1] = -1;
                    mbar_arrive(&tile_full[wg ^ 1]);
                    break;
                }
                tile_slot[wg] = u;
                mbar_arrive(&tile_full[wg]);
                const int m0 = (u / num_n_tiles) * TC_BLOCK_M, n0 = (u % num_n_tiles) * TC_BLOCK_N;
                for (int kb = 0; kb < num_k_blocks; ++kb) {
                    // the next tile is claimed with this one's last k-block: the atomic's round trip runs under the wait for a
                    // free stage, and a CTA claims no more than one tile ahead of the loads it has issued
                    if (kb == num_k_blocks - 1) u = (int)atomicAdd(p.queue, 1u);
                    mbar_wait(&empty_bar[stage], phase ^ 1);              // the warpgroup that consumed this stage has left it
                    uint8_t *st = smem + stage * TC_STAGE_BYTES;
                    mbar_arrive_expect_tx(&full_bar[stage], ((p.dbg & 4) ? 0u : 2 * TC_A_BYTES) + ((p.dbg & 2) ? 0u : 2 * TC_W_BYTES));
                    if (!(p.dbg & 4)) {
                        tma_load_2d(&tm_a_hi, &full_bar[stage], st, kb * TC_BLOCK_K, m0);
                        tma_load_2d(&tm_a_lo, &full_bar[stage], st + TC_A_BYTES, kb * TC_BLOCK_K, m0);
                    }
                    if (!(p.dbg & 2)) {
                        tma_load_2d(&tm_w_hi, &full_bar[stage], st + 2 * TC_A_BYTES, kb * TC_BLOCK_K, n0);
                        tma_load_2d(&tm_w_lo, &full_bar[stage], st + 2 * TC_A_BYTES + TC_W_BYTES, kb * TC_BLOCK_K, n0);
                    }
                    if (++stage == TC_STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== MMA (registers) -> epilogue -> swizzled smem staging -> TMA store =====================
        // Row-strided global stores straight from the accumulator fragments would write 16-byte pieces of 1 KB rows, so
        // each 64 x 64 chunk is staged in shared memory in the SWIZZLE_128B image of the output box (16-byte piece j of
        // row r sits in slot j ^ (r & 7): conflict-free) and one thread per warpgroup hands it to the TMA unit: full
        // 128-byte lines, rows past M clipped by the tensor map.
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int wg = warp >> 2;
        const int rr0 = (warp & 3) * 16 + (lane >> 2);             // fragment rows rr0, rr0 + 8 of each 64-row fragment
        const int q2 = 2 * (lane & 3);                              // fragment column pair within each 8-column group
        const bool has_bias = (p.mode != 1);
        const float slope = (p.mode == 0) ? 0.2f : 1.0f, gain = (p.mode == 0) ? 1.41421356237309515f : 1.0f;
        const float inv_wscale = __ldg(p.inv_wscale);
        uint8_t *stg = staging + wg * (2 * TC_BOX_BYTES);
        const bool storer = ((threadIdx.x & 127) == 0);
        const bool to_f32 = (p.out_f32 != nullptr);
        bool ovf = false;
        float acc0[64], acc1[64];                                    // rows [0, 64) and [64, 128) of the tile
#pragma unroll
        for (int j = 0; j < 64; ++j) { acc0[j] = 0.f; acc1[j] = 0.f; }

        // rows [mrow, mrow + 64) x columns [c0, c0 + 64) of the tile (fragment indices ib .. ib + 31 of `acc`) -> staging -> TMA store
        auto store_chunk = [&](const float (&acc)[64], const int ib, const int mrow, const int n0, const int c0) {
            if (storer) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // staging has been read out
            asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
#pragma unroll
            for (int g = 0; g < 8; ++g) {                           // 8-column group g of the chunk
                const int col = n0 + c0 + 8 * g + q2;
                float2 b = make_float2(0.f, 0.f);
                if (has_bias && col < p.N_total) b = __ldg(reinterpret_cast<const float2 *>(p.bias + col));
#pragma unroll
                for (int h = 0; h < 2; ++h) {                       // fragment rows rr0, rr0 + 8
                    const int rr = rr0 + 8 * h;
                    float f[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        // one instruction stream for the three modes (a per-element branch on p.mode is slow):
                        // no bias = + 0, no activation = slope 1, gain 1 -- exact in fp32
                        float x = __fmul_rn(acc[ib + 4 * g + 2 * h + e], inv_wscale) + (e ? b.y : b.x);
                        x = (x >= 0.f) ? x : __fmul_rn(x, slope);
                        f[e] = __fmul_rn(gain, x);
                    }
                    uint8_t *row = stg + rr * 128;
                    const uint32_t sw = (uint32_t)(rr & 7);
                    if (to_f32) {                                   // columns [0,32) -> box 0, [32,64) -> box 1; 4 floats per piece
                        const int cb = (8 * g + q2) & 31;
                        *reinterpret_cast<float2 *>(row + (g >> 2) * TC_BOX_BYTES + ((((uint32_t)cb >> 2) ^ sw) << 4) + (cb & 3) * 4) =
                            make_float2(f[0], f[1]);
                    } else {                                        // 8 fp16 per 16-byte piece: piece g, bytes [2 q2, 2 q2 + 4)
                        uint32_t hi, lo;
                        split2(f[0], f[1], hi, lo);
                        ovf |= (fabsf(f[0]) > 60000.f) | (fabsf(f[1]) > 60000.f);
                        *reinterpret_cast<uint32_t *>(row + (((uint32_t)g ^ sw) << 4) + 2 * q2) = hi;
                        *reinterpret_cast<uint32_t *>(row + TC_BOX_BYTES + (((uint32_t)g ^ sw) << 4) + 2 * q2) = lo;
                    }
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");          // generic-proxy writes -> visible to the TMA unit
            asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
            if (storer && !(p.dbg & 1) && n0 + c0 < p.N_total) {
                if (to_f32) {
                    tma_store_2d(&tm_o0, stg, n0 + c0, mrow);
                    if (n0 + c0 + 32 < p.N_total) tma_store_2d(&tm_o0, stg + TC_BOX_BYTES, n0 + c0 + 32, mrow);
                } else {
                    tma_store_2d(&tm_o0, stg, n0 + c0, mrow);
                    tma_store_2d(&tm_o1, stg + TC_BOX_BYTES, n0 + c0, mrow);
                }
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        };

        // the CTA's i-th unit (i = 2 j + wg) is this warpgroup's j-th tile; the producer fills the ring with the CTA's k-blocks
        // in order, so k-block kb of unit i is the CTA's k-block i num_k_blocks + kb, which fixes its stage and phase
        for (int i = wg;; i += 2) {
            mbar_wait(&tile_full[wg], (uint32_t)(i >> 1) & 1);
            const int u = tile_slot[wg];
            __syncwarp();
            if (lane == 0) mbar_arrive(&tile_empty[wg]);
            if (u < 0) break;
            const int m0 = (u / num_n_tiles) * TC_BLOCK_M, n0 = (u % num_n_tiles) * TC_BLOCK_N;
            const int g0 = i * num_k_blocks;
            int stage = g0 % TC_STAGES, prev = stage;
            uint32_t phase = (uint32_t)(g0 / TC_STAGES) & 1;
            // ping-pong: the main loop starts once the other warpgroup has issued all MMAs of unit i - 1 (its (i - 1) / 2-th
            // hand-over), so the two main loops alternate on the tensor cores instead of interleaving
            if (i > 0) mbar_wait(&turn_bar[wg], (uint32_t)((i - 1) >> 1) & 1);
            for (int kb = 0; kb < num_k_blocks; ++kb) {
                mbar_wait(&full_bar[stage], phase);                // TMA bytes have landed
                if (!(p.dbg & 8)) {
                    const uint32_t st = smem_u32(smem + stage * TC_STAGE_BYTES);
                    const uint32_t sw = st + 2 * TC_A_BYTES;
                    const uint64_t d_wh = sw128_kmajor_desc(sw), d_wl = sw128_kmajor_desc(sw + TC_W_BYTES);
                    wgmma_fence();
                    split_kblock_m64n128(acc0, sw128_kmajor_desc(st), sw128_kmajor_desc(st + TC_A_BYTES), d_wh, d_wl, kb > 0);
                    split_kblock_m64n128(acc1, sw128_kmajor_desc(st + TC_A_BYTES / 2),
                                         sw128_kmajor_desc(st + TC_A_BYTES + TC_A_BYTES / 2), d_wh, d_wl, kb > 0);
                    wgmma_commit();
                }
                wgmma_wait_1();                                     // k-block kb - 1's MMAs have completed ...
                if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[prev]);   // ... so its smem slot is free
                if (kb == num_k_blocks - 1 && lane == 0) mbar_arrive(&turn_bar[wg ^ 1]);   // hand the tensor cores over
                prev = stage;
                if (++stage == TC_STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait_all();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            store_chunk(acc0, 0, m0, n0, 0);
            store_chunk(acc0, 32, m0, n0, 64);
            store_chunk(acc1, 0, m0 + TC_FRAG_ROWS, n0, 0);
            store_chunk(acc1, 32, m0 + TC_FRAG_ROWS, n0, 64);
        }
        if (ovf) atomicOr(p.overflow, 1u);
        if (storer) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");     // all output boxes are in global memory
    }
}

// ---- operand preparation ------------------------------------------------------------------------------
// PixelNorm (model.py:14-19) + split into fp16 hi/lo.  One warp per row.
__global__ void pixelnorm_split_kernel(const float *__restrict__ x, __half *__restrict__ hi, __half *__restrict__ lo,
                                       int64_t n, int dim, int do_norm, unsigned *overflow) {
    int64_t row = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n) return;
    const int lane = threadIdx.x & 31;
    const float4 *xr = reinterpret_cast<const float4 *>(x + row * dim);
    float r = 1.f;
    if (do_norm) {
        float s = 0.f;
        for (int i = lane; i < dim / 4; i += 32) {
            float4 v = xr[i];
            s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
        }
        s = warp_sum(s);
        r = 1.0f / sqrtf(s / (float)dim + 1e-8f);
    }
    bool ovf = false;
    for (int i = lane; i < dim / 4; i += 32) {
        float4 v = xr[i];
        const float f[4] = {v.x * r, v.y * r, v.z * r, v.w * r};
        tc::store_split4(f, hi, lo, row * dim + 4 * i, ovf);
    }
    if (ovf) atomicOr(overflow, 1u);
}

// ---- weight operand (tc_split_weight) ------------------------------------------------------------------------------
__global__ void weight_absmax_kernel(const float *__restrict__ x, int64_t count, float scale, float *__restrict__ out) {
    float m = 0.f;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
        m = fmaxf(m, fabsf(x[i] * scale));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int *>(out), __float_as_int(m));   // m >= 0: int order == float order
}

// scal[2] = absmax -> scal[1] = 2^s, scal[0] = 2^-s with the largest |w 2^s| in [8192, 16384)
__global__ void pick_wscale_kernel(float *__restrict__ scal) {
    float m = scal[2];
    if (!(m > 0.f)) m = 1.f;
    int e = 0;
    frexpf(m, &e);                         // m = f * 2^e, f in [0.5, 1)
    scal[1] = ldexpf(1.f, 14 - e);
    scal[0] = ldexpf(1.f, e - 14);
}

// one thread per (row, col) of W [rows, cols, taps]: w' = (scale W) 2^s (a power of two: exact) -> fp16 hi / lo at row
// tap' rows + row, i.e. element tap' rows cols + idx; wsq[idx] = the fmaf chain of (scale W)^2 over the taps in order
__global__ void weight_split_kernel(const float *__restrict__ W, int64_t total, int taps, float scale, int reverse,
                                    const float *__restrict__ scal, __half *__restrict__ hi, __half *__restrict__ lo,
                                    float *__restrict__ wsq) {
    const float ws = scal[1];
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        float sq = 0.f;
        for (int t = 0; t < taps; ++t) {
            const float w = W[idx * taps + t] * scale;
            sq = fmaf(w, w, sq);
            const int64_t o = (int64_t)(reverse ? taps - 1 - t : t) * total + idx;
            tc::split1(w * ws, hi[o], lo[o]);
        }
        if (wsq) wsq[idx] = sq;
    }
}

// ---- host side ------------------------------------------------------------------------------------------
// 2-D row-major [rows, cols] fp16 or fp32 tensor, box = box_rows x 128 bytes of a row, 128B swizzle (rows / cols smaller than
// the box are fine: the TMA unit fills the rest of the box with zeros)
static int make_tmap(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols, uint32_t box_rows,
                     CUtensorMapDataType type = CU_TENSOR_MAP_DATA_TYPE_FLOAT16) {
    const uint32_t esize = (type == CU_TENSOR_MAP_DATA_TYPE_FLOAT32) ? 4 : 2;
    const uint64_t dims[2] = {cols, rows};
    const uint64_t strides[1] = {cols * esize};
    const uint32_t box[2] = {128 / esize, box_rows};
    return tc_make_tmap(map, type, base, 2, dims, strides, box);
}

// Tensor-core packed layout (appended after the fp32 SIMT pack inside the same allocation):
//   [n_layers][dim*dim] fp16 W_hi | [n_layers][dim*dim] fp16 W_lo | [n_layers][3] float {inv_wscale, wscale, absmax} | flag
size_t mapping_tc_packed_bytes(int n_layers, int dim) {
    return align_up((size_t)n_layers * dim * dim * 2, 256) * 2 + align_up((size_t)3 * n_layers * sizeof(float), 256) + 256;
}

struct TcPackView {
    __half *w_hi, *w_lo;
    float *scal;              // [n_layers][3], tc_split_weight's {inv_wscale, wscale, absmax}
    unsigned *overflow;
};
static TcPackView tc_pack_view(void *base, int n_layers, int dim) {
    TcPackView v;
    char *p = reinterpret_cast<char *>(base);
    size_t wb = align_up((size_t)n_layers * dim * dim * 2, 256);
    v.w_hi = reinterpret_cast<__half *>(p);
    v.w_lo = reinterpret_cast<__half *>(p + wb);
    v.scal = reinterpret_cast<float *>(p + 2 * wb);
    v.overflow = reinterpret_cast<unsigned *>(p + 2 * wb + align_up((size_t)3 * n_layers * sizeof(float), 256));
    return v;
}

// Splits the already scale-multiplied fp32 weights `pw` ([n_layers][dim*dim]); stream-ordered, no host sync.
int mapping_tc_pack(const float *pw, int n_layers, int dim, void *tc_base, cudaStream_t st) {
    TcPackView v = tc_pack_view(tc_base, n_layers, dim);
    GSB_CHECK_CUDA(cudaMemsetAsync(v.scal, 0, (size_t)3 * n_layers * sizeof(float), st));
    GSB_CHECK_CUDA(cudaMemsetAsync(v.overflow, 0, sizeof(unsigned), st));
    const int64_t per = (int64_t)dim * dim;
    for (int l = 0; l < n_layers; ++l)
        if (int r = tc_split_weight(pw + l * per, dim, dim, 1, 1.0f, false, dim, v.w_hi + l * per, v.w_lo + l * per, v.scal + 3 * l,
                                    nullptr, st)) return r;
    return GSB_OK;
}

int tc_split_weight(const float *w, int rows, int cols, int taps, float scale, bool reverse_taps, int n_pad, __half *hi, __half *lo,
                    float *scal, float *wsq, cudaStream_t st) {
    const int64_t tap_rows = (int64_t)taps * rows, total = (int64_t)rows * cols;
    GSB_CHECK_ARG(w && hi && lo && scal && rows > 0 && cols > 0 && taps > 0 && n_pad >= tap_rows && n_pad % 32 == 0,
                  "tc_split_weight: bad shape (rows=%d cols=%d taps=%d n_pad=%d)", rows, cols, taps, n_pad);
    if (n_pad > tap_rows) {
        const size_t pad_bytes = (size_t)(n_pad - tap_rows) * cols * sizeof(__half);
        GSB_CHECK_CUDA(cudaMemsetAsync(hi + tap_rows * cols, 0, pad_bytes, st));
        GSB_CHECK_CUDA(cudaMemsetAsync(lo + tap_rows * cols, 0, pad_bytes, st));
    }
    weight_absmax_kernel<<<256, 256, 0, st>>>(w, total * taps, scale, scal + 2);
    GSB_CHECK_LAUNCH();
    pick_wscale_kernel<<<1, 1, 0, st>>>(scal);
    GSB_CHECK_LAUNCH();
    weight_split_kernel<<<1024, 256, 0, st>>>(w, total, taps, scale, reverse_taps ? 1 : 0, scal, hi, lo, wsq);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// one launch of the layer kernel over all output tiles; A and W tensor maps must have been built with box rows 128
// `queue`: one unsigned of device memory, zeroed here (stream-ordered), that no concurrent launch uses
static int tc_launch_layer(const CUtensorMap &tm_ah, const CUtensorMap &tm_al, const CUtensorMap &tm_wh, const CUtensorMap &tm_wl,
                           TcParams p, unsigned *queue, int leave_free_sms, cudaStream_t st) {
    // output boxes of the epilogue's TMA stores (64 rows: one accumulator fragment, half of the tile): fp16 hi / lo [M, N]
    // (the next layer's A operand) or fp32 [M, N]
    CUtensorMap tm_o0, tm_o1;
    if (p.out_f32) {
        if (int r = make_tmap(&tm_o0, p.out_f32, (uint64_t)p.M, (uint64_t)p.N_total, TC_FRAG_ROWS,
                              CU_TENSOR_MAP_DATA_TYPE_FLOAT32))
            return r;
        tm_o1 = tm_o0;
    } else {
        if (int r = make_tmap(&tm_o0, p.out_hi, (uint64_t)p.M, (uint64_t)p.N_total, TC_FRAG_ROWS)) return r;
        if (int r = make_tmap(&tm_o1, p.out_lo, (uint64_t)p.M, (uint64_t)p.N_total, TC_FRAG_ROWS)) return r;
    }
    const int m_tiles = (p.M + TC_BLOCK_M - 1) / TC_BLOCK_M, n_tiles = (p.N_total + TC_BLOCK_N - 1) / TC_BLOCK_N;
    int avail = num_sms() - leave_free_sms;
    if (avail < 16) avail = 16;
    if (avail > num_sms()) avail = num_sms();
    {
        static int dbg = -1;
        if (dbg < 0) { const char *e = getenv("GANSPACE_B200_MAPPING_DBG"); dbg = e ? atoi(e) : 0; }
        p.dbg = dbg;
    }
    // work units: single 128 x 128 tiles, two consumer warpgroups per CTA
    const int64_t units = (int64_t)m_tiles * n_tiles;
    GSB_CHECK_ARG(units < (1ll << 31) - 1024, "mapping_layer_tc: too many tiles");
    GSB_CHECK_CUDA(cudaMemsetAsync(queue, 0, sizeof(unsigned), st));
    p.queue = queue;
    const int grid = units < avail ? (int)units : avail;
    mapping_layer_tc_kernel<<<grid, TC_THREADS, TC_SMEM_BYTES, st>>>(tm_ah, tm_al, tm_wh, tm_wl, tm_o0, tm_o1, p);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// out[M, N] (fp32, row-major) = (A_hi + A_lo)[M, K] * (W_hi + W_lo)[N, K]^T * inv_wscale   -- the same persistent
// tensor-core kernel with the plain epilogue.  Both operands are K-major fp16 hi/lo pairs; N % 32 == 0, K % 8 == 0 (the TMA
// unit zero-fills the operand boxes of a ragged last N or K tile and clips its stores).
// Used by the modulated-convolution path (synthesis.cu): one dense contraction per 3x3 tap.
int tc_gemm_plain(const __half *a_hi, const __half *a_lo, int64_t M, int K, const __half *w_hi, const __half *w_lo, int N,
                  const float *inv_wscale, float *out, unsigned *overflow, unsigned *queue, int leave_free_sms, cudaStream_t st) {
    GSB_CHECK_ARG(N % 32 == 0 && N >= 32 && K % 8 == 0 && K >= 8 && M > 0 && M < (1ll << 31) && queue,
                  "tc_gemm_plain: need N%%32==0, K%%8==0 (M=%lld N=%d K=%d)", (long long)M, N, K);
    if (int r = raise_dyn_smem(mapping_layer_tc_kernel, TC_SMEM_BYTES)) return r;
    CUtensorMap tm_ah, tm_al, tm_wh, tm_wl;
    if (int r = make_tmap(&tm_ah, a_hi, (uint64_t)M, (uint64_t)K, TC_BLOCK_M)) return r;
    if (int r = make_tmap(&tm_al, a_lo, (uint64_t)M, (uint64_t)K, TC_BLOCK_M)) return r;
    if (int r = make_tmap(&tm_wh, w_hi, (uint64_t)N, (uint64_t)K, TC_BLOCK_N)) return r;
    if (int r = make_tmap(&tm_wl, w_lo, (uint64_t)N, (uint64_t)K, TC_BLOCK_N)) return r;
    TcParams p;
    p.bias = nullptr; p.out_hi = nullptr; p.out_lo = nullptr; p.out_f32 = out; p.overflow = overflow;
    p.inv_wscale = inv_wscale; p.M = (int)M; p.N_total = N; p.K = K; p.mode = 1;
    return tc_launch_layer(tm_ah, tm_al, tm_wh, tm_wl, p, queue, leave_free_sms, st);
}

// y[n, N] = x[n, K] W[N, K]^T + bias (optionally sqrt2 * lrelu) on the tensor cores, fp32-grade (hi/lo split of both operands
// done here: W per call -- N*K elements, negligible next to the n*N*K product for n >= 128).  N % 256 == 0, K % 64 == 0.
// Used for BigGAN's generator.gen_z (biggan model.py:211-212,232): [B, 256] x [256, 32768].
// ws layout: x_hi, x_lo [n*K] fp16 | w_hi, w_lo [N*K] fp16 | {inv_wscale, wscale, absmax} | overflow flag, tile queue
size_t tc_linear_workspace_bytes(int64_t n, int N, int K) {
    return 2 * align_up((size_t)n * K * 2, 256) + 2 * align_up((size_t)N * K * 2, 256) + 512;
}

int tc_linear(const float *x, const float *w, const float *bias, float *y, int64_t n, int N, int K, bool lrelu, void *ws,
              cudaStream_t st) {
    GSB_CHECK_ARG(N % 256 == 0 && K % TC_BLOCK_K == 0 && n > 0 && n < (1ll << 31) && bias, "tc_linear: need N%%256==0, K%%64==0, bias");
    if (int r = raise_dyn_smem(mapping_layer_tc_kernel, TC_SMEM_BYTES)) return r;
    char *p0 = reinterpret_cast<char *>(ws);
    const size_t xb = align_up((size_t)n * K * 2, 256), wb = align_up((size_t)N * K * 2, 256);
    __half *x_hi = (__half *)p0, *x_lo = (__half *)(p0 + xb), *w_hi = (__half *)(p0 + 2 * xb), *w_lo = (__half *)(p0 + 2 * xb + wb);
    float *scal = (float *)(p0 + 2 * xb + 2 * wb);              // inv_wscale, wscale, absmax
    unsigned *overflow = (unsigned *)(p0 + 2 * xb + 2 * wb + 256);
    GSB_CHECK_CUDA(cudaMemsetAsync(scal, 0, 512, st));
    if (int r = tc_split_weight(w, N, K, 1, 1.0f, false, N, w_hi, w_lo, scal, nullptr, st)) return r;
    pixelnorm_split_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(x, x_hi, x_lo, n, K, 0, overflow);
    GSB_CHECK_LAUNCH();
    CUtensorMap tm_ah, tm_al, tm_wh, tm_wl;
    if (int r = make_tmap(&tm_ah, x_hi, (uint64_t)n, (uint64_t)K, TC_BLOCK_M)) return r;
    if (int r = make_tmap(&tm_al, x_lo, (uint64_t)n, (uint64_t)K, TC_BLOCK_M)) return r;
    if (int r = make_tmap(&tm_wh, w_hi, (uint64_t)N, (uint64_t)K, TC_BLOCK_N)) return r;
    if (int r = make_tmap(&tm_wl, w_lo, (uint64_t)N, (uint64_t)K, TC_BLOCK_N)) return r;
    TcParams p;
    p.bias = bias; p.out_hi = nullptr; p.out_lo = nullptr; p.out_f32 = y; p.overflow = overflow;
    p.inv_wscale = scal; p.M = (int)n; p.N_total = N; p.K = K; p.mode = lrelu ? 0 : 2;
    return tc_launch_layer(tm_ah, tm_al, tm_wh, tm_wl, p, overflow + 1, 0, st);
}

// Full mapping network on the tensor cores.  ws: 4 fp16 buffers of n*dim (two hi/lo ping-pong pairs) + the tile queue.
int mapping_forward_tc(const float *pb, void *tc_base, int n_layers, int dim,
                       const float *d_z, float *d_w, int64_t n, bool pixelnorm, void *ws, int leave_free_sms,
                       cudaStream_t st) {
    GSB_CHECK_ARG(dim % 256 == 0 && dim % TC_BLOCK_K == 0, "mapping_forward_tc: dim must be a multiple of 256");
    GSB_CHECK_ARG(n < (1ll << 31), "mapping_forward_tc: too many rows");
    TcPackView v = tc_pack_view(tc_base, n_layers, dim);
    const size_t buf = align_up((size_t)n * dim * 2, 256);
    __half *a_hi[2] = {reinterpret_cast<__half *>(ws), reinterpret_cast<__half *>((char *)ws + 2 * buf)};
    __half *a_lo[2] = {reinterpret_cast<__half *>((char *)ws + buf), reinterpret_cast<__half *>((char *)ws + 3 * buf)};
    unsigned *queue = reinterpret_cast<unsigned *>((char *)ws + 4 * buf);

    if (int r = raise_dyn_smem(mapping_layer_tc_kernel, TC_SMEM_BYTES)) return r;
    pixelnorm_split_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(d_z, a_hi[0], a_lo[0], n, dim, pixelnorm ? 1 : 0,
                                                                  v.overflow);
    GSB_CHECK_LAUNCH();
    // persistent CTAs, one per SM; `leave_free_sms` keeps some SMs idle for a concurrent latency-critical stream (the IPCA
    // chain's 16-CTA cluster kernels), which otherwise wait for a whole layer launch to drain
    const int64_t per = (int64_t)dim * dim;
    for (int l = 0; l < n_layers; ++l) {
        const int src = l & 1, dst = src ^ 1;
        CUtensorMap tm_ah, tm_al, tm_wh, tm_wl;
        if (int r = make_tmap(&tm_ah, a_hi[src], (uint64_t)n, dim, TC_BLOCK_M)) return r;
        if (int r = make_tmap(&tm_al, a_lo[src], (uint64_t)n, dim, TC_BLOCK_M)) return r;
        if (int r = make_tmap(&tm_wh, v.w_hi + l * per, dim, dim, TC_BLOCK_N)) return r;
        if (int r = make_tmap(&tm_wl, v.w_lo + l * per, dim, dim, TC_BLOCK_N)) return r;
        TcParams p;
        p.bias = pb + (int64_t)l * dim;
        const bool last = (l == n_layers - 1);
        p.out_hi = last ? nullptr : a_hi[dst];
        p.out_lo = last ? nullptr : a_lo[dst];
        p.out_f32 = last ? d_w : nullptr;
        p.overflow = v.overflow;
        p.inv_wscale = v.scal + 3 * l;
        p.M = (int)n; p.N_total = dim; p.K = dim; p.mode = 0;
        if (int r = tc_launch_layer(tm_ah, tm_al, tm_wh, tm_wl, p, queue, leave_free_sms, st)) return r;
    }
    return GSB_OK;
}

size_t mapping_tc_workspace_bytes(int64_t n, int dim) { return 4 * align_up((size_t)n * dim * 2, 256) + 256; }

unsigned *mapping_tc_overflow_flag(void *tc_base, int n_layers, int dim) {
    return tc_pack_view(tc_base, n_layers, dim).overflow;
}

}  // namespace gsb
