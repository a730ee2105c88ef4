// bf16 GEMM for every nn.Linear / conv-as-GEMM on the AF3 path, written for sm_90a (H100):
//   out[tok, feat] = epilogue( sum_k X[tok, k] * W[feat, k] )        (both operands K-major = nn.Linear layout)
// Replaces the cuBLASLt calls behind  F.linear / F.conv1d  in the reference path
// ([O] AF3M:111-114,141,153-154,204-205,343-344,398-402; Q2M:41-43,46-48,199-202,474-475).
//
// Design (one persistent CTA per SM, 9 warps, warp-specialised):
//   warp 8      TMA producer: cp.async.bulk.tensor 2-D loads of 128B-swizzled [rows x 64] bf16 tiles into a
//               STAGES-deep smem ring, completion on mbarriers.
//   warps 0-7   two consumer warpgroups: wgmma.mma_async (m64 x BN x 16, bf16 -> fp32 in registers) straight from the
//               ring with smem descriptors, one k-block group kept in flight; each warpgroup owns 64 of the tile's 128
//               rows.  The finished accumulator goes to an fp32 tile in shared memory, from which the epilogue warps
//               (4 or 8 of them, one row per lane) apply bias / GELU(erf) / residual / SwiGLU with the reference's bf16
//               rounding points and store with TMA or vectorised global stores.
// "Row operand" = the matrix whose rows are the wgmma M dimension (128 per tile), "col operand" = the one whose rows
// are N (BN).  Normal mode: rows = tokens, cols = features.  Swap mode (few tokens, decode):
// rows = weight features (so every wgmma streams weight rows), cols = tokens, and the epilogue writes the
// transposed tile.  Tile order is grouped (GROUP_R row tiles share a col tile) so the 50 MB L2 holds the
// working set of one wave and HBM sees each operand ~once.
#include "common.h"
#include "gemm_epi.h"
#include "ptx.cuh"

#include <cstdlib>

namespace af3 {

struct GemmArgs {
    int R, C, K;  // extents of row operand, col operand, reduction
    int num_r_tiles, num_c_tiles, group_r;
    int n_tok, n_feat;  // logical output extents (features after SwiGLU halving)
    void* out;
    int ldo;
    const bf16* bias;
    const bf16* resid;
    int ld_res;
    int res_period;  // residual row = tok % res_period (positional-embedding add); 0 = plain
    int flags;
    // split-K (swap mode only): each output tile is computed by k_splits CTAs over disjoint K ranges; partial fp32
    // tiles go to `ws`, the CTA that arrives last (per-tile counter) sums them in split order (deterministic) and
    // runs the fused epilogue.  Fills the 132 SMs when the weight matrix has only 28-36 row tiles (decode step).
    // EPI_ROPE (few-token q/k/v projection of the decode step, one 128-row tile = one head): rotary embedding and the
    // KV-cache append are applied in the epilogue ([O] Q2M:100-146, CACHE:119-120) -- q heads go to `out`, k / v heads
    // straight into the cache at slot *rope_pos.
    const float2* rope_cs;   // [n_tok][64] (cos, sin), bf16-rounded
    bf16* k_cache;
    bf16* v_cache;
    const int* rope_pos;     // device int: cache slot of this step
    int rope_H, rope_Hkv, rope_Tmax;
    int tma_epi;    // normal mode: stage the output tile in smem and write it with TMA (coalesced); residual via TMA too
    // SwiGLU weight layout: 0 = gate / up interleaved in blocks of 128 rows (af3_pack_gate_up); > 0 = plain concatenation
    // [gate (n_feat rows); up (n_feat rows)], the value being the first up row -- the two 128-row halves of a tile are then fetched
    // by two TMA boxes, and gate_proj.weight / up_proj.weight can simply be VIEWS of the fused matrix (no second copy in HBM)
    int swiglu_up_row0;
    int k_splits;
    float* ws;      // [tiles][k_splits][BN][128] fp32
    int* counters;  // [tiles], zero on entry, reset to zero by the reducing CTA
    unsigned long long* trace;  // in-graph timeline slot of this launch (common.h) or nullptr
};

constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle atom row
constexpr int GEMM_THREADS = 288;  // warps 0-7: two consumer warpgroups (wgmma + epilogue), warp 8: TMA producer

template <int BN, int NA, int STAGES, bool SWAP>
struct GemmCfg {
    static constexpr int R_BYTES = 128 * NA * BK * 2;
    static constexpr int C_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = R_BYTES + C_BYTES;
    static constexpr int ACC_COLS = NA * BN;
    // the finished fp32 accumulator tile [128 rows][ACC_COLS], handed from the wgmma registers to the epilogue warps
    static constexpr int ACC_BYTES = 128 * ACC_COLS * 4;
    // normal mode: 4 epilogue warps x 2 buffers x (32 rows x 128 B) staging for the TMA-store epilogue
    // swap mode: one [32 tokens x 128 features] bf16 tile to transpose the accumulator for token-major vector I/O
    static constexpr int EPI_STAGE_BYTES = SWAP ? 32 * 128 * 2 : 4 * 2 * 4096;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + EPI_STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert((2 * STAGES + 8) * 8 + 16 <= 256, "barrier area");
    static_assert(BN == 32 || BN == 128, "BN: wgmma shapes m64n32 / m64n128");
    static_assert(SMEM_BYTES <= 232448, "shared memory per CTA");
};

// fp32 accumulator tile in shared memory: 16-byte chunks of row r are XOR-swizzled by r % 8, so that both the fragment stores
// of the warpgroups and the row reads of the epilogue (one row per lane) spread over all banks
template <int COLS>
__device__ __forceinline__ int acc_idx(int r, int c) {
    return r * COLS + ((((c >> 2) ^ (r & 7)) << 2) | (c & 3));
}
// 32 consecutive fp32 columns of row r (c % 4 == 0), as raw bits
template <int COLS>
__device__ __forceinline__ void acc_ld32(const float* buf, int r, int c, uint32_t (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float4 f = *reinterpret_cast<const float4*>(buf + acc_idx<COLS>(r, c + 4 * j));
        v[4 * j] = __float_as_uint(f.x);
        v[4 * j + 1] = __float_as_uint(f.y);
        v[4 * j + 2] = __float_as_uint(f.z);
        v[4 * j + 3] = __float_as_uint(f.w);
    }
}

__device__ __forceinline__ void tile_coords(int t, const GemmArgs& a, int& r, int& c) {
    const int per_group = a.group_r * a.num_c_tiles;
    const int g = t / per_group;
    const int rem = t - g * per_group;
    const int r0 = g * a.group_r;
    const int gr = min(a.group_r, a.num_r_tiles - r0);
    c = rem / gr;
    r = r0 + (rem - c * gr);
}

// epilogue math for one output element; x is the fp32 accumulator
__device__ __forceinline__ float epi_elem(float x, int flags, float bias, float res) {
    if (flags & EPI_BIAS) x += bias;
    x = bf16_round(x);  // nn.Linear output is bf16
    if (flags & EPI_GELU) x = bf16_round(gelu_erf(x));
    if (flags & EPI_RESID) x = bf16_round(x + res);
    return x;
}
__device__ __forceinline__ float epi_swiglu(float g, float u) {
    g = bf16_round(g);
    u = bf16_round(u);
    const float s = bf16_round(g / (1.0f + __expf(-g)));  // F.silu in bf16: fp32 math, one rounding
    return bf16_round(s * u);
}

// EPI >= 0: epilogue flags fixed at compile time (no per-element branches, full ILP across the 32-column chunk);
// EPI < 0: generic instantiation reading a.flags at run time (odd layouts / unusual flag mixes).
// EW = epilogue warps (4 or 8) among the 8 consumer warps.  With 8 (normal mode, epilogues without a TMA-prefetched residual) two
// warps share each 32-row quarter of the tile and split its 64-column groups between them: twice the issue slots for epilogue
// math, which is what bounds short-K GEMMs with expensive epilogues (K = 1280 + GELU: erff per element).
template <int BN, int NA, int STAGES, bool SWAP, int EPI, int EW>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap map_r, const __grid_constant__ CUtensorMap map_c,
            const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_res, const GemmArgs a) {
    using Cfg = GemmCfg<BN, NA, STAGES, SWAP>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    float* accbuf = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint8_t* epi_stage = smem + STAGES * Cfg::STAGE_BYTES + Cfg::ACC_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(epi_stage + Cfg::EPI_STAGE_BYTES);
    uint64_t* empty = full + STAGES;
    uint64_t* rbar = empty + STAGES;  // [4 warps][2 buffers] residual-tile arrival
    uint32_t* flag_slot = reinterpret_cast<uint32_t*>(rbar + 8);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) trace_mark(a.trace, 0);
    const int flags = (EPI >= 0) ? EPI : a.flags;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&map_r);
        tma_prefetch_desc(&map_c);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 8);  // one arrival per consumer warp
        }
        for (int i = 0; i < 8; ++i) mbar_init(&rbar[i], 1);
        if (a.tma_epi) {
            tma_prefetch_desc(&map_out);
            if ((flags & EPI_RESID) && a.res_period == 0) tma_prefetch_desc(&map_res);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();  // the next kernel may start its prologue / weight prefetch behind us

    const int k_splits = SWAP ? a.k_splits : 1;
    const int num_tiles = a.num_r_tiles * a.num_c_tiles * k_splits;  // work items: (tile, split), split fastest
    const int k_blocks_total = (a.K + BK - 1) / BK;
    // K range of split s: blocks [kb_lo(s), kb_lo(s+1)), sizes differ by at most one
    auto kb_lo = [&](int s) { return (s * k_blocks_total) / k_splits; };
    // row of the col operand where the 64 gate rows (normal-mode SwiGLU tile c: output features [64c, 64c + 64)) start; the 64 up
    // rows follow 128 rows later (gate / up interleaved in blocks of 128 rows) or at swiglu_up_row0 + 64c ([gate; up])
    auto gate_row = [&](int c) { return a.swiglu_up_row0 ? c * 64 : (c >> 1) * 256 + (c & 1) * 64; };
    auto up_row = [&](int c) { return a.swiglu_up_row0 ? a.swiglu_up_row0 + c * 64 : gate_row(c) + 128; };

    if (warp == 8) {
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            // Swap mode: the row operand is a WEIGHT matrix, independent of earlier kernels -> its first STAGES tiles are
            // requested before pdl_wait(), so weight streaming overlaps the tail of the previous kernel(s).
            int prefetched = 0;
            if constexpr (SWAP) {
                const int t0 = blockIdx.x;
                if (t0 < num_tiles) {
                    int r, c;
                    tile_coords(t0 / k_splits, a, r, c);
                    const int sp = t0 % k_splits;
                    for (int kb = kb_lo(sp); kb < kb_lo(sp + 1) && prefetched < STAGES; ++kb, ++prefetched) {
                        mbar_arrive_expect_tx(&full[prefetched], Cfg::STAGE_BYTES);
                        uint8_t* sR = smem + prefetched * Cfg::STAGE_BYTES;
#pragma unroll
                        for (int na = 0; na < NA; ++na)
                            tma_load_2d(sR + na * 128 * BK * 2, &map_r, &full[prefetched], kb * BK,
                                        a.swiglu_up_row0 ? na * a.swiglu_up_row0 + r * 128 : (r * NA + na) * 128);
                    }
                }
            }
            pdl_wait();
            int issued = 0;  // k-blocks issued so far by this CTA (the first `prefetched` already have their weights in flight)
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                int r, c;
                tile_coords(t / k_splits, a, r, c);
                const int sp = t % k_splits;
                for (int kb = kb_lo(sp); kb < kb_lo(sp + 1); ++kb, ++issued) {
                    uint8_t* sR = smem + stage * Cfg::STAGE_BYTES;
                    uint8_t* sC = sR + Cfg::R_BYTES;
                    if (issued >= prefetched) {
                        mbar_wait(&empty[stage], phase ^ 1);
                        mbar_arrive_expect_tx(&full[stage], Cfg::STAGE_BYTES);
#pragma unroll
                        for (int na = 0; na < NA; ++na)
                            tma_load_2d(sR + na * 128 * BK * 2, &map_r, &full[stage], kb * BK,
                                        (SWAP && a.swiglu_up_row0) ? na * a.swiglu_up_row0 + r * 128 : (r * NA + na) * 128);
                    }
                    if (!SWAP && (flags & EPI_SWIGLU)) {   // 64 gate rows, then the 64 up rows of the same output features
                        tma_load_2d(sC, &map_c, &full[stage], kb * BK, gate_row(c));
                        tma_load_2d(sC + 64 * BK * 2, &map_c, &full[stage], kb * BK, up_row(c));
                    } else {
                        tma_load_2d(sC, &map_c, &full[stage], kb * BK, c * BN);
                    }
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
        __syncwarp();
    } else {
        // ---- consumer warpgroups: warpgroup wg computes rows [64 wg, 64 wg + 64) of every 128-row block of the row operand with
        //      wgmma (accumulator in registers), hands the finished tile to the epilogue through accbuf, then runs the epilogue
        const int wg = warp >> 2;
        const int tw = threadIdx.x & 127;   // thread within the warpgroup
        const int q = warp & 3;             // 32-row quarter of the tile this warp's epilogue owns
        [[maybe_unused]] const int ehalf = (EW == 8) ? wg : 0;  // which half of the column groups (EW == 8)
        const int row_in_tile = q * 32 + lane;
        const bool epi_warp = warp < EW;
        pdl_wait();  // residual reads / output writes / split-K workspace are ordered after every earlier kernel
        if (threadIdx.x == 0) trace_mark(a.trace, 1);
        int stage = 0;
        uint32_t phase = 0;
        uint32_t egrp = 0;             // running 64-column group counter of this warp (selects the staging buffer)
        uint32_t rpar0 = 0, rpar1 = 0;  // residual-barrier parities per buffer
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            {
                const int sp = t % k_splits;
                const int kb0 = kb_lo(sp), kb1 = kb_lo(sp + 1);
                float accr[NA][BN / 2];
#pragma unroll
                for (int na = 0; na < NA; ++na)
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) accr[na][i] = 0.f;
                int prev = -1;
                for (int kb = kb0; kb < kb1; ++kb) {
                    mbar_wait(&full[stage], phase);
                    const uint32_t sR = smem_u32(smem + stage * Cfg::STAGE_BYTES);
                    const uint32_t sC = sR + Cfg::R_BYTES;
#pragma unroll
                    for (int na = 0; na < NA; ++na) fence_regs(accr[na]);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < BK / 16; ++k) {
                        const uint64_t bdesc = make_smem_desc_sw128(sC + k * 32, 0, 1024);
#pragma unroll
                        for (int na = 0; na < NA; ++na) {
                            const uint64_t adesc = make_smem_desc_sw128(sR + na * 128 * BK * 2 + wg * 64 * 128 + k * 32, 0, 1024);
                            if constexpr (BN == 128)
                                wgmma_m64n128_ss<0, 0>(accr[na], adesc, bdesc, 1);
                            else
                                wgmma_m64n32_ss<0, 0>(accr[na], adesc, bdesc, 1);
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<1>();  // the previous k-block's group has retired: its stage goes back to the producer
#pragma unroll
                    for (int na = 0; na < NA; ++na) fence_regs(accr[na]);
                    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
                    prev = stage;
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
                wgmma_wait<0>();
#pragma unroll
                for (int na = 0; na < NA; ++na) fence_regs(accr[na]);
                if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
                asm volatile("bar.sync 3, 256;" ::: "memory");  // the previous tile's epilogue is done with accbuf
#pragma unroll
                for (int na = 0; na < NA; ++na)
#pragma unroll
                    for (int i = 0; i < BN / 2; i += 2)
                        *reinterpret_cast<float2*>(accbuf + acc_idx<Cfg::ACC_COLS>(wg * 64 + frag_row(tw, i), na * BN + frag_col(tw, i))) =
                            make_float2(accr[na][i], accr[na][i + 1]);
                asm volatile("bar.sync 3, 256;" ::: "memory");
            }
            if (!epi_warp) continue;
            int r, c;
            tile_coords(t / k_splits, a, r, c);
            [[maybe_unused]] const bool swiglu = flags & EPI_SWIGLU;
            [[maybe_unused]] const bool tma_res = a.tma_epi && (flags & EPI_RESID) && a.res_period == 0;
            [[maybe_unused]] const int out_col_base = c * (swiglu ? BN / 2 : BN);
            [[maybe_unused]] const int row0 = r * 128 + q * 32;
            if constexpr (!SWAP) {
                if (tma_res && lane == 0) {  // prefetch the residual slab of group 0 while the accumulator is still in flight
                    bulk_wait_read<0>();
                    const int b0 = egrp & 1;
                    mbar_arrive_expect_tx(&rbar[q * 2 + b0], 4096);
                    tma_load_2d(epi_stage + (q * 2 + b0) * 4096, &map_res, &rbar[q * 2 + b0], out_col_base, row0);
                }
            }
            // few-token mode with a fused residual: this thread's residual vectors of the transposed epilogue (token et / 4,
            // features (et % 4) * 32 ...) do not depend on this GEMM -- request them now, they arrive while the weights stream
            // (the epilogue otherwise exposes one more L2 round trip in the split-K tail)
            [[maybe_unused]] uint4 rv_pre[4];
            [[maybe_unused]] bool rv_ok = false;
            if constexpr (SWAP && BN == 32 && NA == 1) {
                if ((flags & EPI_RESID) && !(flags & EPI_F32OUT) && (a.ldo & 7) == 0 && (a.ld_res & 7) == 0 && a.res_period == 0) {
                    const int et = threadIdx.x;
                    const int tok = c * BN + (et >> 2);
                    const int f0 = r * 128 + (et & 3) * 32;
                    if (tok < a.n_tok) {
                        rv_ok = true;
                        const uint4* rp = reinterpret_cast<const uint4*>(a.resid + static_cast<size_t>(tok) * a.ld_res + f0);
#pragma unroll
                        for (int g4 = 0; g4 < 4; ++g4) rv_pre[g4] = (f0 + g4 * 8 < a.n_feat) ? __ldcg(rp + g4) : make_uint4(0, 0, 0, 0);
                    }
                }
            }
            if (threadIdx.x == 0) trace_mark(a.trace, 2);

            if constexpr (!SWAP) {
                const int tok = r * 128 + row_in_tile;
                const bool row_ok = tok < a.n_tok;
                const int res_row = (a.res_period > 0) ? (tok % a.res_period) : tok;
                if (a.tma_epi) {
                    // ---- smem-staged epilogue: per warp, 64 output columns at a time -> [32 rows x 128 B] swizzled slab -> TMA store
                    const int n_groups = (swiglu ? BN / 2 : BN) / 64;
                    // EW == 8: this warp owns half of the groups and ONE staging buffer (index ehalf); EW == 4: all groups,
                    // two alternating buffers
                    const int g_lo = (EW == 8) ? ehalf * (n_groups / 2) : 0;
                    const int g_hi = (EW == 8) ? g_lo + n_groups / 2 : n_groups;
#pragma unroll 1
                    for (int gi = g_lo; gi < g_hi; ++gi) {
                        const int buf = (EW == 8) ? ehalf : (egrp & 1);
                        uint8_t* sbuf = epi_stage + (q * 2 + buf) * 4096;
                        if (out_col_base + gi * 64 >= a.n_feat) break;  // fully out-of-range group (warp-uniform)
                        if (lane == 0) {
                            if (tma_res) {
                                bulk_wait_read<0>();  // store of the previous group has drained its buffer
                                if (gi + 1 < n_groups && out_col_base + (gi + 1) * 64 < a.n_feat) {
                                    mbar_arrive_expect_tx(&rbar[q * 2 + (buf ^ 1)], 4096);
                                    tma_load_2d(epi_stage + (q * 2 + (buf ^ 1)) * 4096, &map_res, &rbar[q * 2 + (buf ^ 1)],
                                                out_col_base + (gi + 1) * 64, row0);
                                }
                            } else if (EW == 8) {
                                bulk_wait_read<0>();  // single buffer per warp: the previous store has drained it
                            } else {
                                bulk_wait_read<1>();  // the store that last used THIS buffer has drained it
                            }
                        }
                        __syncwarp();
                        if (tma_res) {
                            mbar_wait(&rbar[q * 2 + buf], buf ? rpar1 : rpar0);
                            if (buf) rpar1 ^= 1; else rpar0 ^= 1;
                        }
                        uint8_t* srow = sbuf + lane * 128;
#pragma unroll
                        for (int half = 0; half < 2; ++half) {
                            const int tcol = gi * 64 + half * 32;
                            uint32_t v[32], u[32];
                            acc_ld32<Cfg::ACC_COLS>(accbuf, row_in_tile, tcol, v);
                            if (swiglu) acc_ld32<Cfg::ACC_COLS>(accbuf, row_in_tile, BN / 2 + tcol, u);
                            const int f0 = out_col_base + tcol;
                            float x[32];
                            if (swiglu) {
#pragma unroll
                                for (int j = 0; j < 32; ++j) x[j] = epi_swiglu(__uint_as_float(v[j]), __uint_as_float(u[j]));
                            } else {
                                float bsv[32], rs[32];
                                if ((flags & EPI_BIAS) && f0 + 32 <= a.n_feat) {
                                    const uint4* bp = reinterpret_cast<const uint4*>(a.bias + f0);
#pragma unroll
                                    for (int j = 0; j < 4; ++j) {
                                        uint4 bv = __ldg(bp + j);
                                        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&bv);
#pragma unroll
                                        for (int e = 0; e < 4; ++e) {
                                            float2 f = __bfloat1622float2(h[e]);
                                            bsv[j * 8 + e * 2] = f.x;
                                            bsv[j * 8 + e * 2 + 1] = f.y;
                                        }
                                    }
                                } else {
#pragma unroll
                                    for (int j = 0; j < 32; ++j)
                                        bsv[j] = ((flags & EPI_BIAS) && f0 + j < a.n_feat) ? __bfloat162float(a.bias[f0 + j]) : 0.f;
                                }
                                if (tma_res) {
#pragma unroll
                                    for (int g4 = 0; g4 < 4; ++g4) {
                                        const uint4 rv = *reinterpret_cast<const uint4*>(srow + (((half * 4 + g4) ^ (lane & 7)) << 4));
                                        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&rv);
#pragma unroll
                                        for (int e = 0; e < 4; ++e) {
                                            float2 f = __bfloat1622float2(h[e]);
                                            rs[g4 * 8 + e * 2] = f.x;
                                            rs[g4 * 8 + e * 2 + 1] = f.y;
                                        }
                                    }
                                } else if (flags & EPI_RESID) {  // periodic residual (positional embedding): direct loads
                                    const bf16* rp = a.resid + static_cast<size_t>(res_row) * a.ld_res + f0;
#pragma unroll
                                    for (int j = 0; j < 32; ++j) rs[j] = (row_ok && f0 + j < a.n_feat) ? __bfloat162float(rp[j]) : 0.f;
                                } else {
#pragma unroll
                                    for (int j = 0; j < 32; ++j) rs[j] = 0.f;
                                }
#pragma unroll
                                for (int j = 0; j < 32; ++j) x[j] = epi_elem(__uint_as_float(v[j]), flags, bsv[j], rs[j]);
                            }
#pragma unroll
                            for (int g4 = 0; g4 < 4; ++g4)
                                *reinterpret_cast<uint4*>(srow + (((half * 4 + g4) ^ (lane & 7)) << 4)) =
                                    make_uint4(pack_bf16x2(x[8 * g4], x[8 * g4 + 1]), pack_bf16x2(x[8 * g4 + 2], x[8 * g4 + 3]),
                                               pack_bf16x2(x[8 * g4 + 4], x[8 * g4 + 5]), pack_bf16x2(x[8 * g4 + 6], x[8 * g4 + 7]));
                        }
                        fence_proxy_async_smem();
                        __syncwarp();
                        if (lane == 0) {
                            tma_store_2d(&map_out, sbuf, out_col_base + gi * 64, row0);
                            bulk_commit();
                        }
                        ++egrp;
                    }
                } else if (flags & EPI_SWIGLU) {
                    // cols [0, BN/2) = gate, [BN/2, BN) = up of the same BN/2 output features
                    constexpr int HALF = BN / 2;
#pragma unroll 1
                    for (int ch = 0; ch < HALF / 32; ++ch) {
                        uint32_t g[32], u[32];
                        acc_ld32<Cfg::ACC_COLS>(accbuf, row_in_tile, ch * 32, g);
                        acc_ld32<Cfg::ACC_COLS>(accbuf, row_in_tile, HALF + ch * 32, u);
                        const int f0 = c * HALF + ch * 32;
                        if (row_ok && f0 < a.n_feat) {
                            bf16* o = reinterpret_cast<bf16*>(a.out) + static_cast<size_t>(tok) * a.ldo + f0;
                            if (f0 + 32 <= a.n_feat && (a.ldo & 7) == 0) {
                                uint32_t w[16];
#pragma unroll
                                for (int j = 0; j < 16; ++j)
                                    w[j] = pack_bf16x2(epi_swiglu(__uint_as_float(g[2 * j]), __uint_as_float(u[2 * j])),
                                                       epi_swiglu(__uint_as_float(g[2 * j + 1]), __uint_as_float(u[2 * j + 1])));
#pragma unroll
                                for (int j = 0; j < 4; ++j)
                                    reinterpret_cast<uint4*>(o)[j] = make_uint4(w[4 * j], w[4 * j + 1], w[4 * j + 2], w[4 * j + 3]);
                            } else {
                                _Pragma("unroll") for (int j = 0; j < 32; ++j) if (f0 + j < a.n_feat)
                                    o[j] = __float2bfloat16_rn(epi_swiglu(__uint_as_float(g[j]), __uint_as_float(u[j])));
                            }
                        }
                    }
                } else {
#pragma unroll 1
                    for (int ch = 0; ch < BN / 32; ++ch) {
                        uint32_t v[32];
                        acc_ld32<Cfg::ACC_COLS>(accbuf, row_in_tile, ch * 32, v);
                        const int f0 = c * BN + ch * 32;
                        if (row_ok && f0 < a.n_feat) {
                            const bool fullv = (f0 + 32 <= a.n_feat);
                            float x[32];
                            if (fullv && (flags & EPI_BIAS)) {
                                const uint4* bp = reinterpret_cast<const uint4*>(a.bias + f0);
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    uint4 bv = __ldg(bp + j);
                                    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&bv);
#pragma unroll
                                    for (int e = 0; e < 4; ++e) {
                                        float2 f = __bfloat1622float2(h[e]);
                                        x[j * 8 + e * 2] = f.x;
                                        x[j * 8 + e * 2 + 1] = f.y;
                                    }
                                }
                            } else {
#pragma unroll
                                for (int j = 0; j < 32; ++j)
                                    x[j] = ((flags & EPI_BIAS) && f0 + j < a.n_feat) ? __bfloat162float(a.bias[f0 + j]) : 0.f;
                            }
                            float rs[32];
                            if (flags & EPI_RESID) {
                                const bf16* rp = a.resid + static_cast<size_t>(res_row) * a.ld_res + f0;
                                if (fullv && (a.ld_res & 7) == 0) {
#pragma unroll
                                    for (int j = 0; j < 4; ++j) {
                                        uint4 rv = *(reinterpret_cast<const uint4*>(rp) + j);
                                        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&rv);
#pragma unroll
                                        for (int e = 0; e < 4; ++e) {
                                            float2 f = __bfloat1622float2(h[e]);
                                            rs[j * 8 + e * 2] = f.x;
                                            rs[j * 8 + e * 2 + 1] = f.y;
                                        }
                                    }
                                } else {
#pragma unroll
                                    for (int j = 0; j < 32; ++j) rs[j] = (f0 + j < a.n_feat) ? __bfloat162float(rp[j]) : 0.f;
                                }
                            } else {
#pragma unroll
                                for (int j = 0; j < 32; ++j) rs[j] = 0.f;
                            }
#pragma unroll
                            for (int j = 0; j < 32; ++j) x[j] = epi_elem(__uint_as_float(v[j]), flags, x[j], rs[j]);

                            if (flags & EPI_F32OUT) {
                                float* o = reinterpret_cast<float*>(a.out) + static_cast<size_t>(tok) * a.ldo + f0;
                                if (fullv && (a.ldo & 3) == 0) {
#pragma unroll
                                    for (int j = 0; j < 8; ++j)
                                        reinterpret_cast<float4*>(o)[j] = make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
                                } else {
                                    _Pragma("unroll") for (int j = 0; j < 32; ++j) if (f0 + j < a.n_feat) o[j] = x[j];
                                }
                            } else {
                                bf16* o = reinterpret_cast<bf16*>(a.out) + static_cast<size_t>(tok) * a.ldo + f0;
                                if (fullv && (a.ldo & 7) == 0) {
#pragma unroll
                                    for (int j = 0; j < 4; ++j)
                                        reinterpret_cast<uint4*>(o)[j] =
                                            make_uint4(pack_bf16x2(x[8 * j], x[8 * j + 1]), pack_bf16x2(x[8 * j + 2], x[8 * j + 3]),
                                                       pack_bf16x2(x[8 * j + 4], x[8 * j + 5]), pack_bf16x2(x[8 * j + 6], x[8 * j + 7]));
                                } else {
                                    _Pragma("unroll") for (int j = 0; j < 32; ++j) if (f0 + j < a.n_feat) o[j] = __float2bfloat16_rn(x[j]);
                                }
                            }
                        }
                    }
                }
            } else {
                // swapped: accumulator row = output feature, column = token
                const int feat = r * 128 + row_in_tile;
                const bool feat_ok = feat < a.n_feat;
                const float bias = ((flags & EPI_BIAS) && feat_ok) ? __bfloat162float(a.bias[feat]) : 0.f;
#pragma unroll 1
                for (int ch = 0; ch < BN / 32; ++ch) {
                    uint32_t v[32], u[32];
                    acc_ld32<Cfg::ACC_COLS>(accbuf, row_in_tile, ch * 32, v);
                    if constexpr (NA == 2) acc_ld32<Cfg::ACC_COLS>(accbuf, row_in_tile, BN + ch * 32, u);
                    if constexpr (NA == 1 && BN == 32) {
                        if (k_splits > 1) {
                            // publish this split's partial tile: ws[tile][split][col][row] (row fastest: coalesced)
                            const int tile = t / k_splits, sp = t % k_splits;
                            float* wt = a.ws + (static_cast<size_t>(tile) * k_splits) * (BN * 128);
#pragma unroll
                            for (int j = 0; j < 32; ++j) wt[(sp * BN + j) * 128 + row_in_tile] = __uint_as_float(v[j]);
                            // release: the barrier orders every thread's partial stores before thread 64's fence + counter
                            // increment (fences are cumulative -- the cooperative-groups grid-sync pattern); acquire: thread 64's
                            // fence after the increment, then the barrier, then L2 (.cg) loads by everyone
                            asm volatile("bar.sync 1, 128;" ::: "memory");
                            if (threadIdx.x == 0) {
                                __threadfence();
                                const int arrived_now = atomicAdd(a.counters + tile, 1);
                                __threadfence();
                                *reinterpret_cast<volatile int*>(flag_slot) = arrived_now;
                            }
                            asm volatile("bar.sync 1, 128;" ::: "memory");
                            const int arrived = *reinterpret_cast<volatile int*>(flag_slot);
                            if (arrived != k_splits - 1) continue;  // not the last split of this tile: done
                            // Sum in split order (deterministic: 0, 1, 2, ...).  Two register buffers keep the loads of split s + 1
                            // (and s + 2) in flight while split s is added: k_splits dependent L2 round trips become ~k_splits / 2.
                            float sum[32], ta[32], tb[32];
                            auto ld_part = [&](float (&d)[32], int s2) {
#pragma unroll
                                for (int j = 0; j < 32; ++j) d[j] = __ldcg(wt + (s2 * BN + j) * 128 + row_in_tile);
                            };
                            ld_part(ta, 0);
#pragma unroll
                            for (int j = 0; j < 32; ++j) sum[j] = 0.f;
                            for (int s2 = 0; s2 < k_splits; s2 += 2) {
                                if (s2 + 1 < k_splits) ld_part(tb, s2 + 1);
#pragma unroll
                                for (int j = 0; j < 32; ++j) sum[j] += ta[j];
                                if (s2 + 2 < k_splits) ld_part(ta, s2 + 2);
                                if (s2 + 1 < k_splits) {
#pragma unroll
                                    for (int j = 0; j < 32; ++j) sum[j] += tb[j];
                                }
                            }
#pragma unroll
                            for (int j = 0; j < 32; ++j) v[j] = __float_as_uint(sum[j]);
                            if (threadIdx.x == 0) a.counters[tile] = 0;
                        }
                    }
                    const int tok0 = c * BN + ch * 32;
                    if constexpr (BN == 32) {
                        if (!(flags & EPI_F32OUT) && (a.ldo & 7) == 0 && (!(flags & EPI_RESID) || ((a.ld_res & 7) == 0 && a.res_period == 0))) {
                            // ---- transposed epilogue: this thread owns feature `feat` for 32 tokens, but the output (and the
                            // residual) are token-major.  Pre-residual values go through a [32 tok][128 feat] bf16 smem tile so
                            // that global traffic is 16-byte vectors along the feature dimension (4 loads + 4 stores per thread
                            // instead of 32 + 32 scalar ones whose latencies ptxas otherwise serialises).
                            bf16* tile = reinterpret_cast<bf16*>(epi_stage);
#pragma unroll
                            for (int j = 0; j < 32; ++j) {
                                float y;
                                if constexpr (NA == 2)
                                    y = epi_swiglu(__uint_as_float(v[j]), __uint_as_float(u[j]));
                                else
                                    y = epi_elem(__uint_as_float(v[j]), flags & ~EPI_RESID, bias, 0.f);
                                tile[j * 128 + row_in_tile] = __float2bfloat16_rn(y);
                            }
                            asm volatile("bar.sync 2, 128;" ::: "memory");
                            const int et = threadIdx.x;             // 0..127 within the epilogue warps
                            const int tok = tok0 + (et >> 2);
                            const int f0 = r * 128 + (et & 3) * 32;      // first of this thread's 32 features
                            if ((flags & EPI_ROPE) && tok < a.n_tok) {
                                // tile r = head r of the fused projection: [0,H) query, [H,H+Hkv) key, then value heads
                                const int head = r, q4 = et & 3;
                                const uint4* tp = reinterpret_cast<const uint4*>(tile + (et >> 2) * 128 + q4 * 32);
                                bf16* op;
                                bool store = true;
                                if (head < a.rope_H)
                                    op = reinterpret_cast<bf16*>(a.out) + static_cast<size_t>(tok) * a.ldo + f0;
                                else {
                                    const int hk = (head - a.rope_H) % a.rope_Hkv;
                                    bf16* cache = (head < a.rope_H + a.rope_Hkv) ? a.k_cache : a.v_cache;
                                    const int slot = *a.rope_pos;
                                    // a full cache must never be written past its allocation (the host raises before launching;
                                    // this guards graph replays whose position lives on the device)
                                    store = slot >= 0 && slot < a.rope_Tmax;
                                    op = cache + ((static_cast<size_t>(tok) * a.rope_Hkv + hk) * a.rope_Tmax + (store ? slot : 0)) * 128 + q4 * 32;
                                }
                                if (!store) {
                                } else if (head < a.rope_H + a.rope_Hkv) {
                                    const uint4* pp = reinterpret_cast<const uint4*>(tile + (et >> 2) * 128 + (q4 ^ 2) * 32);  // d +- 64
                                    const float2* cs = a.rope_cs + static_cast<size_t>(tok) * 64 + (q4 & 1) * 32;
                                    const float sgn = (q4 < 2) ? -1.f : 1.f;  // rotate_half: -x[d+64] for d < 64, +x[d-64] otherwise
#pragma unroll
                                    for (int g4 = 0; g4 < 4; ++g4) {
                                        const uint4 xv = tp[g4], pv = pp[g4];
                                        const __nv_bfloat162* xh = reinterpret_cast<const __nv_bfloat162*>(&xv);
                                        const __nv_bfloat162* ph = reinterpret_cast<const __nv_bfloat162*>(&pv);
                                        uint32_t o4[4];
#pragma unroll
                                        for (int e = 0; e < 4; ++e) {
                                            const float2 xf = __bfloat1622float2(xh[e]), pf = __bfloat1622float2(ph[e]);
                                            const float2 c0 = __ldg(cs + g4 * 8 + 2 * e), c1 = __ldg(cs + g4 * 8 + 2 * e + 1);
                                            const float o0 = bf16_round(xf.x * c0.x) + bf16_round(sgn * pf.x * c0.y);
                                            const float o1 = bf16_round(xf.y * c1.x) + bf16_round(sgn * pf.y * c1.y);
                                            o4[e] = pack_bf16x2(o0, o1);
                                        }
                                        reinterpret_cast<uint4*>(op)[g4] = make_uint4(o4[0], o4[1], o4[2], o4[3]);
                                    }
                                } else {
#pragma unroll
                                    for (int g4 = 0; g4 < 4; ++g4) reinterpret_cast<uint4*>(op)[g4] = tp[g4];
                                }
                            } else if (!(flags & EPI_ROPE) && tok < a.n_tok) {
                                const uint4* tp = reinterpret_cast<const uint4*>(tile + (et >> 2) * 128 + (et & 3) * 32);
                                bf16* op = reinterpret_cast<bf16*>(a.out) + static_cast<size_t>(tok) * a.ldo + f0;
                                uint4 rv[4];
                                if (flags & EPI_RESID) {
                                    if constexpr (NA == 1) {
                                        if (rv_ok) {   // requested before the accumulator wait (same token / features: ch == 0 for BN = 32)
#pragma unroll
                                            for (int g4 = 0; g4 < 4; ++g4) rv[g4] = rv_pre[g4];
                                        }
                                    } else {
                                        const uint4* rp = reinterpret_cast<const uint4*>(a.resid + static_cast<size_t>(tok) * a.ld_res + f0);
#pragma unroll
                                        for (int g4 = 0; g4 < 4; ++g4)
                                            if (f0 + g4 * 8 < a.n_feat) rv[g4] = __ldcg(rp + g4);
                                    }
                                }
#pragma unroll
                                for (int g4 = 0; g4 < 4; ++g4) {
                                    if (f0 + g4 * 8 < a.n_feat) {   // n_feat is a multiple of 8 on this path (ldo % 8 == 0)
                                        uint4 yv = tp[g4];
                                        if (flags & EPI_RESID) {
                                            const __nv_bfloat162* yh = reinterpret_cast<const __nv_bfloat162*>(&yv);
                                            const __nv_bfloat162* rh = reinterpret_cast<const __nv_bfloat162*>(&rv[g4]);
                                            uint32_t o4[4];
#pragma unroll
                                            for (int e = 0; e < 4; ++e) {
                                                const float2 yf = __bfloat1622float2(yh[e]), rf = __bfloat1622float2(rh[e]);
                                                o4[e] = pack_bf16x2(yf.x + rf.x, yf.y + rf.y);
                                            }
                                            yv = make_uint4(o4[0], o4[1], o4[2], o4[3]);
                                        }
                                        reinterpret_cast<uint4*>(op)[g4] = yv;
                                    }
                                }
                            }
                            asm volatile("bar.sync 2, 128;" ::: "memory");  // tile may be rewritten by the next work item
                            continue;
                        }
                    }
                    if (feat_ok) {
                        float res[32];
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const int tok = tok0 + j;
                            res[j] = 0.f;
                            if (NA == 1 && (flags & EPI_RESID) && tok < a.n_tok) {
                                const int rr = (a.res_period > 0) ? (tok % a.res_period) : tok;
                                res[j] = __bfloat162float(__ldcg(a.resid + static_cast<size_t>(rr) * a.ld_res + feat));
                            }
                        }
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const int tok = tok0 + j;
                            if (tok < a.n_tok) {
                                float x;
                                if constexpr (NA == 2)
                                    x = epi_swiglu(__uint_as_float(v[j]), __uint_as_float(u[j]));
                                else
                                    x = epi_elem(__uint_as_float(v[j]), flags, bias, res[j]);
                                if (flags & EPI_F32OUT)
                                    reinterpret_cast<float*>(a.out)[static_cast<size_t>(tok) * a.ldo + feat] = x;
                                else
                                    reinterpret_cast<bf16*>(a.out)[static_cast<size_t>(tok) * a.ldo + feat] = __float2bfloat16_rn(x);
                            }
                        }
                    }
                }
            }
        }
    }

    if (!SWAP && warp < EW && lane == 0) bulk_wait_read<0>();  // staged tiles must be read out before smem goes away
    __syncthreads();
    if (threadIdx.x == 0) trace_mark(a.trace, 3);
}

template <int BN, int NA, int STAGES, bool SWAP, int EPI, int EW = 4>
static int launch_epi(const CUtensorMap& mr, const CUtensorMap& mc, const CUtensorMap& mo, const CUtensorMap& mres,
                  const GemmArgs& a, cudaStream_t stream) {
    using Cfg = GemmCfg<BN, NA, STAGES, SWAP>;
    auto kern = gemm_kernel<BN, NA, STAGES, SWAP, EPI, EW>;
    static DeviceOnce once;
    if (once.first()) {
        AF3_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    }
    const int tiles = a.num_r_tiles * a.num_c_tiles * (SWAP && a.k_splits > 1 ? a.k_splits : 1);
    const int grid = tiles < sm_count() ? tiles : sm_count();
    AF3_CHECK_CUDA(launch_kernel(kern, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, stream, mr, mc, mo, mres, a));
    return 0;
}

// Host entry.  x: [n_tok, K] bf16 (pitch ldx), w: [n_rows_w, K] bf16 (pitch ldw) where n_rows_w = n_feat, or the
// gate/up-interleaved 2*ceil(n_feat/128)*128 rows when EPI_SWIGLU.  out: [n_tok, n_feat] (pitch ldo).
// compile-time epilogue specialisations for the flag sets the AF3 path uses; anything else -> generic (-1)
template <int BN, int NA, int STAGES, bool SWAP>
static int launch(const CUtensorMap& mr, const CUtensorMap& mc, const CUtensorMap& mo, const CUtensorMap& mres,
                  const GemmArgs& a, cudaStream_t stream) {
#define AF3_EPI_CASE(F) \
    case (F):           \
        return launch_epi<BN, NA, STAGES, SWAP, (F)>(mr, mc, mo, mres, a, stream);
    if constexpr (!SWAP) {
        // 8 epilogue warps where the epilogue (not the MMA) bounds the tile: TMA-store path without a TMA residual
        if (a.tma_epi && !((a.flags & EPI_RESID) && a.res_period == 0)) {
            switch (a.flags) {
                case 0:
                    return launch_epi<BN, NA, STAGES, SWAP, 0, 8>(mr, mc, mo, mres, a, stream);
                case EPI_BIAS:
                    return launch_epi<BN, NA, STAGES, SWAP, EPI_BIAS, 8>(mr, mc, mo, mres, a, stream);
                case EPI_BIAS | EPI_GELU:
                    return launch_epi<BN, NA, STAGES, SWAP, EPI_BIAS | EPI_GELU, 8>(mr, mc, mo, mres, a, stream);
                case EPI_BIAS | EPI_GELU | EPI_RESID:
                    return launch_epi<BN, NA, STAGES, SWAP, EPI_BIAS | EPI_GELU | EPI_RESID, 8>(mr, mc, mo, mres, a, stream);
                default:
                    break;
            }
        }
    }
    if (SWAP || a.tma_epi) {
        switch (a.flags) {
            AF3_EPI_CASE(0)
            AF3_EPI_CASE(EPI_BIAS)
            AF3_EPI_CASE(EPI_BIAS | EPI_GELU)
            AF3_EPI_CASE(EPI_BIAS | EPI_RESID)
            AF3_EPI_CASE(EPI_RESID)
            AF3_EPI_CASE(EPI_SWIGLU)
            AF3_EPI_CASE(EPI_F32OUT)
            AF3_EPI_CASE(EPI_BIAS | EPI_GELU | EPI_RESID)
            AF3_EPI_CASE(EPI_BIAS | EPI_ROPE)
            default:
                break;
        }
    }
#undef AF3_EPI_CASE
    return launch_epi<BN, NA, STAGES, SWAP, -1>(mr, mc, mo, mres, a, stream);
}

size_t gemm_workspace_bytes() { return (8u << 20) + 4096 * sizeof(int); }

int gemm_bf16(cudaStream_t stream, const bf16* x, int ldx, const bf16* w, int ldw, void* out, int ldo, int n_tok,
              int n_feat, int K, int flags, const bf16* bias, const bf16* resid, int ld_res, int res_period,
              void* workspace, size_t workspace_bytes, const RopeEpilogue* rope) {
    AF3_REQUIRE(n_tok > 0 && n_feat > 0 && K > 0, "gemm: empty problem");
    AF3_REQUIRE((K % 8) == 0 && (ldx % 8) == 0 && (ldw % 8) == 0, "gemm: K and pitches must be multiples of 8");
    AF3_REQUIRE(!(flags & EPI_BIAS) || bias, "gemm: bias flag without pointer");
    AF3_REQUIRE(!(flags & EPI_RESID) || resid, "gemm: residual flag without pointer");
    const bool swiglu = flags & EPI_SWIGLU;
    const bool concat = swiglu && (flags & EPI_SWIGLU_CONCAT);
    AF3_REQUIRE(!(flags & EPI_SWIGLU_CONCAT) || (swiglu && n_feat % 128 == 0), "gemm: the [gate; up] layout needs SwiGLU and n_feat % 128 == 0");
    flags &= ~EPI_SWIGLU_CONCAT;
    const int w_rows = swiglu ? 2 * ceil_div(n_feat, 128) * 128 : n_feat;
    GemmArgs a{};
    a.K = K;
    a.n_tok = n_tok;
    a.n_feat = n_feat;
    a.out = out;
    a.ldo = ldo;
    a.bias = bias;
    a.resid = resid;
    a.ld_res = ld_res;
    a.res_period = res_period;
    a.flags = flags;
    a.swiglu_up_row0 = concat ? n_feat : 0;
    a.k_splits = 1;
    a.trace = trace_next_slot();
    if (flags & EPI_ROPE) {
        AF3_REQUIRE(rope && rope->cs && rope->k_cache && rope->v_cache && rope->pos, "gemm: EPI_ROPE needs the rope arguments");
        AF3_REQUIRE(n_tok <= 64 && n_feat == (rope->H + 2 * rope->Hkv) * 128 && (ldo % 8) == 0 && !(flags & (EPI_RESID | EPI_F32OUT | EPI_SWIGLU)),
                    "gemm: EPI_ROPE is the few-token fused q/k/v projection with head_dim 128");
        a.rope_cs = reinterpret_cast<const float2*>(rope->cs);
        a.k_cache = rope->k_cache;
        a.v_cache = rope->v_cache;
        a.rope_pos = rope->pos;
        a.rope_H = rope->H;
        a.rope_Hkv = rope->Hkv;
        a.rope_Tmax = rope->Tmax;
    }
    CUtensorMap mx, mw, mo, mres;
    const bool swap = n_tok <= 64;
    if (!swap) {
        constexpr int BN = 128;
        a.R = n_tok;
        a.C = w_rows;
        a.num_r_tiles = ceil_div(n_tok, 128);
        a.num_c_tiles = ceil_div(w_rows, BN);
        // rasterisation: GROUP_R row tiles stay L2-resident (~20 MB of the 50 MB L2) while the col-operand tiles stream
        // past them, so the streamed operand is re-read num_r_tiles / GROUP_R times instead of once per row tile
        {
            const long long tile_bytes = 128ll * K * 2;
            long long g = (20ll << 20) / tile_bytes;
            a.group_r = static_cast<int>(g < 8 ? 8 : (g > 256 ? 256 : g));
        }
        if (int e = make_tmap_2d(&mx, x, K, n_tok, ldx, BK, 128)) return e;
        if (int e = make_tmap_2d(&mw, w, K, w_rows, ldw, BK, swiglu ? 64 : BN)) return e;
        // smem-staged TMA-store epilogue whenever the output (and residual) layout allows 16-byte-aligned rows
        const bool res_plain = (flags & EPI_RESID) && res_period == 0;
        a.tma_epi = !(flags & EPI_F32OUT) && (ldo % 8 == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0) &&
                    (!res_plain || ((ld_res % 8 == 0) && ((reinterpret_cast<uintptr_t>(resid) & 15) == 0)));
        mo = mx;
        mres = mx;
        if (a.tma_epi) {
            if (int e = make_tmap_2d(&mo, out, n_feat, n_tok, ldo, 64, 32)) return e;
            if (res_plain)
                if (int e = make_tmap_2d(&mres, resid, n_feat, n_tok, ld_res, 64, 32)) return e;
        }
        return launch<BN, 1, 4, false>(mx, mw, mo, mres, a, stream);
    }
    constexpr int BN = 32;
    a.R = w_rows;
    a.C = n_tok;
    a.num_c_tiles = ceil_div(n_tok, BN);
    a.group_r = 1;
    if (int e = make_tmap_2d(&mw, w, K, w_rows, ldw, BK, 128)) return e;
    if (int e = make_tmap_2d(&mx, x, K, n_tok, ldx, BK, BN)) return e;
    // Pipeline depth of the few-token mode: 10 x 20 KB (NA = 1) / 5 x 36 KB (NA = 2) stages, as deep as the 227 KB of shared memory
    // allows next to the accumulator tile: the weight streams of a few-token GEMM are latency-bound on the bytes in flight per SM.
    if (swiglu) {
        a.num_r_tiles = ceil_div(w_rows, 256);
        return launch<BN, 2, 5, true>(mw, mx, mw, mw, a, stream);
    }
    a.num_r_tiles = ceil_div(w_rows, 128);
    // split-K when the tile grid cannot fill the GPU and a (zero-initialised) workspace was supplied
    a.k_splits = 1;
    const int tiles = a.num_r_tiles * a.num_c_tiles;
    const int kb_total = ceil_div(K, BK);
    if (workspace && workspace_bytes >= gemm_workspace_bytes() && tiles * 2 <= sm_count() && tiles <= 4096) {
        int s = sm_count() / tiles;
        const int forced = [] { const char* e = getenv("AF3_KSPLIT"); return e ? atoi(e) : 0; }();  // experiments only (read per call)
        if (forced > 0) s = forced;
        if (s > kb_total / 4) s = kb_total / 4;  // keep at least 4 k-blocks per split
        if (s > 16) s = 16;
        if (s >= 2 && static_cast<size_t>(tiles) * s * BN * 128 * sizeof(float) <= (8u << 20)) {
            a.k_splits = s;
            a.ws = reinterpret_cast<float*>(workspace);
            a.counters = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(workspace) + (8u << 20));
        }
    }
    // ring depth: 10 x 20 KB = 200 KB in flight per SM (the few-token streams are latency-bound on bytes in flight)
    return launch<BN, 1, 10, true>(mw, mx, mw, mw, a, stream);
}

}  // namespace af3
