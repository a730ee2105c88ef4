// bf16 GEMM for every nn.Linear / conv-as-GEMM on the AF3 path, written for sm_90a (H100):
//   out[tok, feat] = epilogue( sum_k X[tok, k] * W[feat, k] )        (both operands K-major = nn.Linear layout)
// Replaces the cuBLASLt calls behind  F.linear / F.conv1d  in the reference path
// ([O] AF3M:111-114,141,153-154,204-205,343-344,398-402; Q2M:41-43,46-48,199-202,474-475).
//
// Three kernels, one persistent CTA per SM each, picked by the token count and, in normal mode, by K and the epilogue:
//
// gemm_tok_wide_kernel (normal mode, K >= 2048, no periodic residual), 3 warpgroups: the producer below, and two consumer
//                  warpgroups that share each 128 x 256 tile (64 token rows each, one m64n256k16 per k16 step, 3 x 48 KB
//                  stages).  Sharing the weight slice cuts the shared-memory operand reads and TMA writes per FLOP that
//                  cap the 128 x 128 tiles; its epilogue is not overlapped, which costs more than it gains at small K.
//
// gemm_tok_kernel (normal mode, n_tok > 64, every other case; rows = tokens, cols = features), 3 warpgroups, ping-pong:
//   warpgroup 0    TMA producer: cp.async.bulk.tensor 2-D loads of 128B-swizzled [rows x 64] bf16 tiles into a
//                  STAGES-deep smem ring, in the CTA's tile order, completion on mbarriers.  Gives its registers to
//                  the consumers (setmaxnreg).
//   warpgroups 1-2 consumers, alternate tiles of the CTA: each owns a whole 128 x 128 output tile (two wgmma
//                  m64n128k16 per k16 step, 128 fp32 accumulators per thread, one k-block group in flight) and runs
//                  the epilogue straight from the accumulator fragments -- bias / GELU(erf) / residual / SwiGLU with the
//                  reference's bf16 rounding points -> stmatrix into a 128B-swizzled bf16 slab -> TMA store.  While
//                  one warpgroup runs its epilogue the other runs its main loop, so the tensor cores stay busy.
//
// gemm_fp8_tok_kernel (FP8 normal mode, n_tok > 64): the wide kernel's layout with e4m3 operands and 128 x 128 tiles; each
//                  k-block is promoted out of the QGMMA accumulator with its block scales (see the kernel).
//
// gemm_kernel (few-token / swap mode, decode), 9 warps:
//   warp 8         TMA producer, as above.
//   warps 0-7      two consumer warpgroups: wgmma.mma_async (m64 x BN x 16) straight from the ring, each warpgroup
//                  owns 64 of the tile's 128 rows.  The finished accumulator goes to an fp32 tile in shared memory,
//                  from which warps 0-3 (one row per lane) run the epilogue and the split-K reduction.
//   "Row operand" = the matrix whose rows are the wgmma M dimension (128 per tile) = weight features (so every wgmma
//   streams weight rows), "col operand" = the tokens (BN = 32); the epilogue writes the transposed tile.
//   With FP8 = true (gemm_fp8, n_tok <= 64) both operands are block-scaled e4m3 and each 128-wide k-block is
//   promoted out of the QGMMA accumulator into fp32 with its scales.
//
// Shared pieces, written once: the ring cursor (Ring), the consumer k-loop of all three kernels (ring_mma / ring_drain),
// and for the two token-major kernels the shared-memory carve-up and prologue (TokSmem, tok_prologue), the producer loop
// (tok_produce; each kernel says how the weight rows of a tile are loaded) and the register epilogue (epi_fragment into
// OutSlabs, which also load the residual and store the tile by TMA).  All are __forceinline__: a call inside a wgmma
// kernel makes ptxas serialise every wgmma (C7510).
//
// Tile order is grouped (GROUP_R row tiles share a col tile) so the 50 MB L2 holds the working set of one wave and
// HBM sees each operand ~once.
#include "common.h"
#include "gemm_epi.h"
#include "ptx.cuh"

#include <cstdlib>

namespace af3 {

struct GemmArgs {
    int K;  // reduction extent
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
    int tma_epi;    // normal mode: stage the output tile in smem and write it with TMA (coalesced); plain residual via TMA too
    // SwiGLU weight layout: 0 = gate / up interleaved in blocks of 128 rows (af3_pack_gate_up); > 0 = plain concatenation
    // [gate (n_feat rows); up (n_feat rows)], the value being the first up row -- the two 128-row halves of a tile are then fetched
    // by two TMA boxes, and gate_proj.weight / up_proj.weight can simply be VIEWS of the fused matrix (no second copy in HBM)
    int swiglu_up_row0;
    int k_splits;
    float* ws;      // [tiles][k_splits][BN][128] fp32
    int* counters;  // [tiles], zero on entry, reset to zero by the reducing CTA
    unsigned long long* trace;  // in-graph timeline slot of this launch (common.h) or nullptr
    // FP8 few-token kernel: activation group scales sx [K/128][n_tok], weight_scale_inv sw [w_rows/128][ld_sw]
    const float* sx;
    const float* sw;
    int ld_sw;
    // EPI_XENT (lm_head_xent): labels [n_tok] (shifted), one (max, sum exp) partial per (token, column tile) at
    // xent_part[tok * num_c_tiles + c], the label's bf16-rounded logit at xent_tgt[tok]
    const int64_t* labels;
    float2* xent_part;
    float* xent_tgt;
};

constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle atom row

template <int V>
struct IntC {
    static constexpr int value = V;
};

// Position in a STAGES-deep smem ring: the stage, and the parity of the mbarrier phase its current use completes.
// Ring slot g (the g-th k-block through the ring) is stage g % STAGES in phase (g / STAGES) & 1.
template <int STAGES>
struct Ring {
    int stage;
    uint32_t phase;
    __device__ __forceinline__ explicit Ring(int g = 0) : stage(g % STAGES), phase((g / STAGES) & 1) {}
    __device__ __forceinline__ void next() {
        if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
        }
    }
};

// Consumer k-loop of every kernel here: n k-blocks from the ring into the accumulators, one k-block group in flight.
// mma(stage) issues the wgmma of one k-block; fence() fences the accumulator registers.  A stage goes back to the producer
// (one arrival per warp) once the group that read it has retired.  Returns the stage still held (-1 when n == 0), which
// ring_drain releases; in between, every full-barrier wait is behind the caller (the ping-pong kernel hands over there).
template <int STAGES, class Mma, class Fence>
__device__ __forceinline__ int ring_mma(Ring<STAGES>& ring, uint64_t* full, uint64_t* empty, int n, Mma&& mma, Fence&& fence) {
    const bool lane0 = (threadIdx.x & 31) == 0;
    int prev = -1;
    for (int kb = 0; kb < n; ++kb) {
        mbar_wait(&full[ring.stage], ring.phase);
        fence();
        wgmma_fence();
        mma(ring.stage);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's group has retired: its stage goes back to the producer
        fence();
        if (prev >= 0 && lane0) mbar_arrive(&empty[prev]);
        prev = ring.stage;
        ring.next();
    }
    return prev;
}
template <class Fence>
__device__ __forceinline__ void ring_drain(uint64_t* empty, int held, Fence&& fence) {
    wgmma_wait<0>();
    fence();
    if (held >= 0 && (threadIdx.x & 31) == 0) mbar_arrive(&empty[held]);
}

// ---- normal mode
constexpr int TOK_THREADS = 384;  // warpgroup 0: TMA producer, warpgroups 1-2: consumers

// Output staging of one consumer warpgroup of a token-major kernel: NS 128B-swizzled bf16 slabs of [ROWS rows][64
// columns], one TMA store each.  A plain residual is TMA-loaded into the same slabs while the main loop runs and read
// back in the accumulator's fragment layout with ldmatrix.
template <int ROWS, int NS>
struct OutSlabs {
    static constexpr int SLAB_BYTES = ROWS * 128;
    static constexpr int BYTES = NS * SLAB_BYTES;
    uint8_t* p;
    // 16-byte chunk (row, column group cg = 8 columns) as a shared-memory address
    __device__ __forceinline__ uint32_t addr(int row, int cg) const {
        return smem_u32(p) + (cg >> 3) * SLAB_BYTES + row * 128 + (((cg & 7) ^ (row & 7)) << 4);
    }
    // leader: residual rows [row0, row0 + ROWS) x the slabs' output columns from col0 that lie below n_feat
    __device__ __forceinline__ void load_res(const CUtensorMap* map_res, uint64_t* bar, int col0, int row0, int n_feat) const {
        bulk_wait_read<0>();  // the previous tile's store has read the slabs
        int ns = 1;
        while (ns < NS && col0 + 64 * ns < n_feat) ++ns;
        mbar_arrive_expect_tx(bar, ns * SLAB_BYTES);
        for (int s = 0; s < ns; ++s) tma_load_2d(p + s * SLAB_BYTES, map_res, bar, col0 + 64 * s, row0);
    }
    // whole warpgroup, before staging: the previous tile's store has read the slabs and the residual (tma_res) has landed
    __device__ __forceinline__ void acquire(bool leader, bool tma_res, int bar_id, uint64_t* res_bar, uint32_t& res_par) const {
        if (!tma_res && leader) bulk_wait_read<0>();
        named_bar_sync(bar_id, 128);
        if (tma_res) {
            mbar_wait(res_bar, res_par);
            res_par ^= 1;
        }
    }
    // whole warpgroup, after staging: the first n slabs (those below n_feat) go out by TMA
    __device__ __forceinline__ void store(bool leader, int bar_id, const CUtensorMap* map_out, int n, int col0, int row0, int n_feat) const {
        fence_proxy_async_smem();
        named_bar_sync(bar_id, 128);
        if (leader) {
            for (int s = 0; s < n; ++s)
                if (col0 + 64 * s < n_feat) tma_store_2d(map_out, p + s * SLAB_BYTES, col0 + 64 * s, row0);
            bulk_commit();
        }
    }
};

template <int STAGES_>
struct TokCfg {
    static constexpr int STAGES = STAGES_;
    static constexpr int KB = BK;                        // K elements per k-block
    static constexpr int X_BYTES = 128 * BK * 2;         // 128 token rows x 64
    static constexpr int STAGE_BYTES = 2 * X_BYTES;      // + 128 weight rows x 64
    using Out = OutSlabs<128, 2>;                        // per consumer warpgroup: the 128 output columns of its tile
    static constexpr int STAGING_BYTES = 2 * Out::BYTES;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert((2 * STAGES + 4) * 8 <= 256, "barrier area");
    static_assert(SMEM_BYTES <= 232448, "shared memory per CTA");
};
// Ring depth, chosen by measurement on an H100 80GB HBM3 (700 W): 4 stages ran the prefill GEMMs 3-10 % faster than 5 (the
// most that fits beside the 64 KB of output slabs) -- e.g. SwiGLU gate/up 24960 x 37888 x 3584 at 618-624 TFLOP/s against
// 572-574 -- while the encoder's K = 1280 GEMMs moved by 1-4 % either way.
constexpr int TOK_STAGES = 4;

template <int STAGES_>
struct WideCfg {
    static constexpr int STAGES = STAGES_;
    static constexpr int KB = BK;
    static constexpr int X_BYTES = 128 * BK * 2;         // 128 token rows x 64
    static constexpr int W_BYTES = 256 * BK * 2;         // 256 weight rows x 64
    static constexpr int STAGE_BYTES = X_BYTES + W_BYTES;
    using Out = OutSlabs<64, 4>;                         // per consumer warpgroup: its 64 x 256 quarter of the tile
    static constexpr int STAGING_BYTES = 2 * Out::BYTES;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert((2 * STAGES + 4) * 8 <= 256, "barrier area");
    static_assert(SMEM_BYTES <= 232448, "shared memory per CTA");
};
// 3 x 48 KB stages + 64 KB of staging (≈ 209 KB), chosen by measurement on an H100 80GB HBM3 (700 W): 4 stages with half
// the staging (two epilogue passes) was as fast within run-to-run spread (prefill GEMMs -1.5 to +5 %, their time-weighted
// sum 0.5 % slower) and needs the second pass.
constexpr int WIDE_STAGES = 3;

// FP8 token-major tiles: 128 tokens x 128 weight rows, one k-block = 128 e4m3 = one 128-byte swizzle row = one scale group
template <int STAGES_>
struct Fp8TokCfg {
    static constexpr int STAGES = STAGES_;
    static constexpr int KB = 128;
    static constexpr int X_BYTES = 128 * 128;            // 128 token rows x 128 e4m3
    static constexpr int STAGE_BYTES = 2 * X_BYTES;      // + 128 weight rows x 128 e4m3
    using Out = OutSlabs<64, 2>;                         // per consumer warpgroup: its 64 x 128 half of the output tile
    static constexpr int STAGING_BYTES = 2 * Out::BYTES;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert((2 * STAGES + 4) * 8 <= 256, "barrier area");
    static_assert(SMEM_BYTES <= 232448, "shared memory per CTA");
};
constexpr int FP8_TOK_STAGES = 6;

// ---- few-token (swap) mode
constexpr int GEMM_THREADS = 288;  // warps 0-7: two consumer warpgroups (wgmma; warps 0-3 also run the epilogue), warp 8: TMA producer

template <int BN, int NA, int STAGES>
struct GemmCfg {
    static constexpr int R_BYTES = 128 * NA * BK * 2;
    static constexpr int C_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = R_BYTES + C_BYTES;
    static constexpr int ACC_COLS = NA * BN;
    // the finished fp32 accumulator tile [128 rows][ACC_COLS], handed from the wgmma registers to the epilogue warps
    static constexpr int ACC_BYTES = 128 * ACC_COLS * 4;
    // one [32 tokens x 128 features] bf16 tile to transpose the accumulator for token-major vector I/O
    static constexpr int EPI_STAGE_BYTES = 32 * 128 * 2;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + EPI_STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(2 * STAGES * 8 + 16 <= 256, "barrier area");
    static_assert(BN == 32, "BN: wgmma shape m64n32");
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

// two consecutive bf16 of a row vector (bias / residual row) as floats; zero from column n on.  vec: p + col is 4-byte aligned
__device__ __forceinline__ float2 ld2(const bf16* p, int col, int n, bool vec) {
    if (vec && col + 1 < n) return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p + col));
    return make_float2(col < n ? __bfloat162float(p[col]) : 0.f, col + 1 < n ? __bfloat162float(p[col + 1]) : 0.f);
}

// ============================================================================ normal mode (n_tok > 64), shared pieces
// Shared memory of the token-major kernels: the ring (1024-byte aligned for the 128B swizzle), the output slabs of both
// consumer warpgroups, then the barriers.
template <class Cfg>
struct TokSmem {
    uint8_t* ring;
    uint8_t* staging;
    uint64_t* full;
    uint64_t* empty;
    uint64_t* rbar;   // [2] residual slabs of consumer 0 / 1 have landed
    uint64_t* order;  // [2] ping-pong kernel only: one completion per main loop of consumer 0 / 1
    __device__ __forceinline__ explicit TokSmem(uint8_t* raw) {
        ring = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
        staging = ring + Cfg::STAGES * Cfg::STAGE_BYTES;
        full = reinterpret_cast<uint64_t*>(staging + Cfg::STAGING_BYTES);
        empty = full + Cfg::STAGES;
        rbar = empty + Cfg::STAGES;
        order = rbar + 2;
    }
};

// Thread 0 of a token-major kernel: descriptor prefetch and barrier init.  `empty` counts empty_arrivals per phase, one
// per warp that reads the stage; the `order` barriers are initialised only when the kernel uses them.
template <class Cfg>
__device__ __forceinline__ void tok_prologue(const TokSmem<Cfg>& sm, uint32_t empty_arrivals, bool order, const GemmArgs& a,
                                             const CUtensorMap* map_x, const CUtensorMap* map_w, const CUtensorMap* map_out,
                                             const CUtensorMap* map_res, bool tma_epi, bool tma_res) {
    trace_mark(a.trace, 0);
    tma_prefetch_desc(map_x);
    tma_prefetch_desc(map_w);
    if (tma_epi) tma_prefetch_desc(map_out);
    if (tma_res) tma_prefetch_desc(map_res);
    for (int i = 0; i < Cfg::STAGES; ++i) {
        mbar_init(&sm.full[i], 1);
        mbar_init(&sm.empty[i], empty_arrivals);
    }
    for (int i = 0; i < 2; ++i) {
        mbar_init(&sm.rbar[i], 1);
        if (order) mbar_init(&sm.order[i], 1);
    }
    fence_barrier_init();
}

// Producer of the token-major kernels: the k-blocks of the CTA's tiles, in tile order, into the ring.  A stage holds the
// tile's 128 token rows of X, then from X_BYTES on its weight rows, which load_w(sW, bar, k0, c) requests for column tile c.
template <class Cfg, class LoadW>
__device__ __forceinline__ void tok_produce(const TokSmem<Cfg>& sm, const CUtensorMap* map_x, const GemmArgs& a, LoadW&& load_w) {
    const int num_tiles = a.num_r_tiles * a.num_c_tiles;
    const int kb_n = (a.K + Cfg::KB - 1) / Cfg::KB;
    Ring<Cfg::STAGES> ring;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int r, c;
        tile_coords(t, a, r, c);
        for (int kb = 0; kb < kb_n; ++kb) {
            uint8_t* sX = sm.ring + ring.stage * Cfg::STAGE_BYTES;
            uint64_t* bar = &sm.full[ring.stage];
            mbar_wait(&sm.empty[ring.stage], ring.phase ^ 1);
            mbar_arrive_expect_tx(bar, Cfg::STAGE_BYTES);
            tma_load_2d(sX, map_x, bar, kb * Cfg::KB, r * 128);
            load_w(sX + Cfg::X_BYTES, bar, kb * Cfg::KB, c);
            ring.next();
        }
    }
}

// Register epilogue of the token-major kernels: one 64-row x N accumulator fragment (wgmma layout: acc[i] at row
// 16 warp + lane / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (lane % 4) + (i & 1)) through epi_elem / epi_swiglu and
// stmatrix into slab rows [srow, srow + 64).  row0 / out_col0: the fragment's first token row and output column.
// SwiGLU: gate in the first, up in the second half of the fragment, N / 2 output columns.
// RES: 0 none, 1 residual already in the slabs (TMA, read back with ldmatrix), 2 rows tok % res_period from global memory.
template <int N, int RES, class Out>
__device__ __forceinline__ void epi_fragment(const float (&acc)[N / 2], const Out& slabs, int srow, int row0, int out_col0, int flags,
                                          const GemmArgs& a) {
    const int tw = threadIdx.x & 127;
    const int warp = tw >> 5, lane = tw & 31;
    const int frow = warp * 16 + (lane >> 2);
    const int fcol = 2 * (lane & 3);
    // stmatrix / ldmatrix x4 over column groups (2 n2, 2 n2 + 1) x rows (+0, +8): this lane addresses row
    // 16 warp + 8 ((lane >> 3) & 1) + lane % 8 of the fragment, column group 2 n2 + (lane >> 4)
    const int mrow = warp * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
    const int mcg = lane >> 4;
    const bool swiglu = flags & EPI_SWIGLU;
    const bool bias_vec = (reinterpret_cast<uintptr_t>(a.bias) & 3) == 0;
    const bool res_vec = (reinterpret_cast<uintptr_t>(a.resid) & 3) == 0 && (a.ld_res & 1) == 0;
    const bf16* rp[2] = {a.resid, a.resid};
    if constexpr (RES == 2) {
        const int rr0 = (row0 + frow) % a.res_period;
        rp[0] += static_cast<size_t>(rr0) * a.ld_res;
        rp[1] += static_cast<size_t>((rr0 + 8) % a.res_period) * a.ld_res;
    }
#pragma unroll
    for (int n2 = 0; n2 < (swiglu ? N / 32 : N / 16); ++n2) {
        const uint32_t maddr = slabs.addr(srow + mrow, 2 * n2 + mcg);
        uint32_t rr[4];
        if constexpr (RES == 1) ldmatrix_x4(maddr, rr);  // residual pairs in the accumulator's fragment layout
        uint32_t y[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int cg = 2 * n2 + (q >> 1);  // column group; q & 1: rows +0 / +8
            const int i = 4 * cg + 2 * (q & 1);
            if (swiglu) {
                y[q] = pack_bf16x2(epi_swiglu(acc[i], acc[i + N / 4]), epi_swiglu(acc[i + 1], acc[i + N / 4 + 1]));
            } else {
                const int col = out_col0 + 8 * cg + fcol;
                const float2 b = (flags & EPI_BIAS) ? ld2(a.bias, col, a.n_feat, bias_vec) : make_float2(0.f, 0.f);
                float2 res = make_float2(0.f, 0.f);
                if constexpr (RES == 1) res = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&rr[q]));
                if constexpr (RES == 2) res = ld2(rp[q & 1], col, a.n_feat, res_vec);
                y[q] = pack_bf16x2(epi_elem(acc[i], flags, b.x, res.x), epi_elem(acc[i + 1], flags, b.y, res.y));
            }
        }
        stmatrix_x4(maddr, y[0], y[1], y[2], y[3]);
    }
}

// Cross-entropy epilogue of the 128 x 128 ping-pong kernel (EPI_XENT): softmax partials of the tile's 128 token rows over its
// 128 columns, straight from the accumulator fragments, after the logits (if any) have been stored.  The accumulators are
// rounded to bf16 in place, as the stored logits are, and set to -inf at columns >= V (exp gives 0).  A row's 128 columns are spread over the 4 lanes of a quad (32 each): (max, sum
// exp(v - max)) per lane, then across the quad; lane 0 of the quad writes the partial.  The lane holding column labels[tok]
// writes that logit: exactly one tile and one lane own a label in [0, V), none owns anything else.  Rows past n_tok (zero
// filled by the TMA load) are skipped.
__device__ __forceinline__ void xent_partials(float (&acc)[2][64], int r, int c, const GemmArgs& a) {
    const int tw = threadIdx.x & 127;
    const int lane = tw & 31;
    const int frow = (tw >> 5) * 16 + (lane >> 2);
    const int fcol = 2 * (lane & 3);
    const int col0 = c * 128;
    const int n_valid = a.n_feat - col0 - fcol;  // columns 8 cg + e of this lane below V: 8 cg + e < n_valid
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            const int tok = r * 128 + h * 64 + frow + 8 * p;
            const bool live = tok < a.n_tok;
            float m = -INFINITY;
#pragma unroll
            for (int cg = 0; cg < 16; ++cg) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float& v = acc[h][4 * cg + 2 * p + e];
                    v = 8 * cg + e < n_valid ? bf16_round(v) : -INFINITY;
                    m = fmaxf(m, v);
                }
            }
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
            float s = 0.f;
#pragma unroll
            for (int cg = 0; cg < 16; ++cg) {
#pragma unroll
                for (int e = 0; e < 2; ++e) s += __expf(acc[h][4 * cg + 2 * p + e] - m);
            }
            // the label's column within the tile, -1 unless it lies in this tile and below V
            const long long lab = live ? a.labels[tok] : -1;
            const int own = (lab >= col0 && lab < col0 + 128 && lab < a.n_feat) ? static_cast<int>(lab - col0) : -1;
            float tgt = 0.f;
#pragma unroll
            for (int cg = 0; cg < 16; ++cg) {
#pragma unroll
                for (int e = 0; e < 2; ++e) tgt = 8 * cg + fcol + e == own ? acc[h][4 * cg + 2 * p + e] : tgt;
            }
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            if (live && (lane & 3) == 0) a.xent_part[static_cast<size_t>(tok) * a.num_c_tiles + c] = make_float2(m, s);
            if (own >= 0 && (own & 7) >> 1 == (lane & 3)) a.xent_tgt[tok] = tgt;
        }
    }
}

// ============================================================================ normal mode, 128 x 128 ping-pong tiles
// EPI >= 0: epilogue flags fixed at compile time (no per-element branches); EPI < 0: generic instantiation reading
// a.flags at run time (odd layouts / unusual flag mixes).
//
// Ring protocol.  The producer fills the ring with the k-blocks of the CTA's tiles in order; the tile with local index j
// (j = 0, 1, ...; global tile blockIdx.x + j * gridDim.x) belongs to consumer warpgroup j % 2, and its k-blocks are ring
// slots j * kb_n ... (j + 1) * kb_n - 1, so each consumer derives stage and phase of its tile and skips the other's.
// mbarrier parity waits are only sound for a waiter at most one phase ahead of the barrier, so the consumers start their
// main loops in tile order: consumer j % 2 begins tile j once the other has issued all of tile j - 1 (barrier `order`).
// That is the ping-pong: the other warpgroup's epilogue overlaps this one's main loop.
template <int STAGES, int EPI>
__global__ void __launch_bounds__(TOK_THREADS, 1)
gemm_tok_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_res, const GemmArgs a) {
    using Cfg = TokCfg<STAGES>;
    extern __shared__ uint8_t smem_raw[];
    const TokSmem<Cfg> sm(smem_raw);

    const int wg = threadIdx.x >> 7;
    const int tw = threadIdx.x & 127;
    const int flags = (EPI >= 0) ? EPI : a.flags;
    const bool swiglu = flags & EPI_SWIGLU;
    const bool tma_res = a.tma_epi && (flags & EPI_RESID) && a.res_period == 0;
    constexpr bool xent = EPI >= 0 && (EPI & EPI_XENT);
    static_assert(!xent || EPI == (EPI_XENT | EPI_F32OUT), "the cross-entropy epilogue stores plain fp32 logits");

    // `empty`: 4 arrivals, one per warp of the warpgroup that consumes the tile; `order` barriers for the ping-pong
    if (threadIdx.x == 0) tok_prologue(sm, 4, true, a, &map_x, &map_w, &map_out, &map_res, a.tma_epi, tma_res);
    __syncthreads();
    pdl_launch_dependents();  // the next kernel may start its prologue behind us

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (tw == 0) {
            pdl_wait();
            tok_produce(sm, &map_x, a, [&](uint8_t* sW, uint64_t* bar, int k0, int c) {
                if (swiglu) {
                    // SwiGLU tile c (output features [64c, 64c + 64)): the 64 gate rows, then the 64 up rows of the same
                    // features -- 128 rows later (gate / up interleaved in blocks of 128 rows) or at swiglu_up_row0 + 64c ([gate; up])
                    const int gate_row = a.swiglu_up_row0 ? c * 64 : (c >> 1) * 256 + (c & 1) * 64;
                    const int up_row = a.swiglu_up_row0 ? a.swiglu_up_row0 + c * 64 : gate_row + 128;
                    tma_load_2d(sW, &map_w, bar, k0, gate_row);
                    tma_load_2d(sW + 64 * BK * 2, &map_w, bar, k0, up_row);
                } else {
                    tma_load_2d(sW, &map_w, bar, k0, c * 128);
                }
            });
        }
    } else {
        setmaxnreg_inc<232>();
        const int cw = wg - 1;  // consumer index
        const bool leader = tw == 0;
        const typename Cfg::Out slabs{sm.staging + cw * Cfg::Out::BYTES};
        const int num_tiles = a.num_r_tiles * a.num_c_tiles;
        const int kb_n = (a.K + BK - 1) / BK;
        pdl_wait();  // residual reads / output writes are ordered after every earlier kernel
        if (threadIdx.x == 128) trace_mark(a.trace, 1);
        uint32_t rpar = 0;
        for (int j = cw;; j += 2) {
            const int t = blockIdx.x + j * gridDim.x;
            if (t >= num_tiles) break;
            int r, c;
            tile_coords(t, a, r, c);
            const int out_col0 = c * (swiglu ? 64 : 128);
            // residual slabs of this tile: they arrive while the main loop runs
            if (tma_res && leader) slabs.load_res(&map_res, &sm.rbar[cw], out_col0, r * 128, a.n_feat);

            // ---- main loop: 128 x 128 tile, two m64n128k16 per k16 step (rows 0-63, rows 64-127)
            float acc[2][64];
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 64; ++i) acc[h][i] = 0.f;
            if (j > 0) mbar_wait(&sm.order[cw ^ 1], ((j - 1) >> 1) & 1);  // tile j - 1 fully issued by the other consumer
            Ring<STAGES> ring(j * kb_n);  // ring slot of this tile's first k-block
            auto fence = [&] {
                fence_regs(acc[0]);
                fence_regs(acc[1]);
            };
            const int held = ring_mma(ring, sm.full, sm.empty, kb_n, [&](int stage) {
                const uint32_t sX = smem_u32(sm.ring + stage * Cfg::STAGE_BYTES);
                const uint32_t sW = sX + Cfg::X_BYTES;
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    const uint64_t bdesc = make_smem_desc_sw128(sW + k * 32, 0, 1024);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        wgmma_m64n128_ss<0, 0>(acc[h], make_smem_desc_sw128(sX + h * 64 * 128 + k * 32, 0, 1024), bdesc, 1);
                }
            }, fence);
            if (leader) mbar_arrive(&sm.order[cw]);  // every full-barrier wait of this tile is behind us: the other consumer may start
            ring_drain(sm.empty, held, fence);
            if (threadIdx.x == 128) trace_mark(a.trace, 2);

            // ---- epilogue from the accumulator fragments
            // the compile-time epilogues are launched only with the TMA-store path (gemm_bf16); the direct-store fallback
            // exists in the generic instantiation alone, which keeps the specialised kernels small.  The cross-entropy
            // epilogue (lm_head_xent) stores the fp32 logits by direct stores when a.out is set, then writes its partials.
            if (!xent && (EPI >= 0 || a.tma_epi)) {
                slabs.acquire(leader, tma_res, 1 + cw, &sm.rbar[cw], rpar);
                // one unrolled pass over the tile per residual source, so that each pass holds only its own operands
                auto stage_tile = [&](auto res_src) {
                    constexpr int RES = decltype(res_src)::value;
                    epi_fragment<128, RES>(acc[0], slabs, 0, r * 128, out_col0, flags, a);
                    epi_fragment<128, RES>(acc[1], slabs, 64, r * 128 + 64, out_col0, flags, a);
                };
                if (tma_res)
                    stage_tile(IntC<1>{});
                else if (flags & EPI_RESID)  // periodic residual (positional embedding)
                    stage_tile(IntC<2>{});
                else
                    stage_tile(IntC<0>{});
                slabs.store(leader, 1 + cw, &map_out, swiglu ? 1 : 2, out_col0, r * 128, a.n_feat);
            } else if (!xent || a.out) {
                // direct stores (output rows not 16-byte aligned, fp32 output): element pairs straight from the fragments
                const int warp = tw >> 5, lane = tw & 31;
                const int frow = warp * 16 + (lane >> 2);
                const int fcol = 2 * (lane & 3);
                const bool bias_vec = (reinterpret_cast<uintptr_t>(a.bias) & 3) == 0;
                const bool res_vec = (reinterpret_cast<uintptr_t>(a.resid) & 3) == 0 && (a.ld_res & 1) == 0;
                const bool out_vec = (reinterpret_cast<uintptr_t>(a.out) & ((flags & EPI_F32OUT) ? 7 : 3)) == 0 && (a.ldo & 1) == 0;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int p = 0; p < 2; ++p) {
                        const int tok = r * 128 + h * 64 + frow + 8 * p;
                        if (tok >= a.n_tok) continue;
                        const int res_row = (a.res_period > 0) ? tok % a.res_period : tok;
#pragma unroll
                        for (int cg = 0; cg < (swiglu ? 8 : 16); ++cg) {
                            const int i = 4 * cg + 2 * p;
                            const int col = out_col0 + 8 * cg + fcol;
                            if (col >= a.n_feat) continue;
                            float2 v;
                            if (swiglu) {
                                v = make_float2(epi_swiglu(acc[h][i], acc[h][i + 32]), epi_swiglu(acc[h][i + 1], acc[h][i + 33]));
                            } else {
                                const float2 b = (flags & EPI_BIAS) ? ld2(a.bias, col, a.n_feat, bias_vec) : make_float2(0.f, 0.f);
                                const float2 res = (flags & EPI_RESID)
                                                       ? ld2(a.resid + static_cast<size_t>(res_row) * a.ld_res, col, a.n_feat, res_vec)
                                                       : make_float2(0.f, 0.f);
                                v = make_float2(epi_elem(acc[h][i], flags, b.x, res.x), epi_elem(acc[h][i + 1], flags, b.y, res.y));
                            }
                            const size_t o = static_cast<size_t>(tok) * a.ldo + col;
                            const bool pair = out_vec && col + 1 < a.n_feat;
                            if (flags & EPI_F32OUT) {
                                float* op = reinterpret_cast<float*>(a.out) + o;
                                if (pair) {
                                    *reinterpret_cast<float2*>(op) = v;
                                } else {
                                    op[0] = v.x;
                                    if (col + 1 < a.n_feat) op[1] = v.y;
                                }
                            } else {
                                bf16* op = reinterpret_cast<bf16*>(a.out) + o;
                                if (pair) {
                                    *reinterpret_cast<uint32_t*>(op) = pack_bf16x2(v.x, v.y);
                                } else {
                                    op[0] = __float2bfloat16_rn(v.x);
                                    if (col + 1 < a.n_feat) op[1] = __float2bfloat16_rn(v.y);
                                }
                            }
                        }
                    }
                }
            }
            if constexpr (xent) xent_partials(acc, r, c, a);  // after the store: the store's temporaries are dead by then
        }
        if (leader) bulk_wait_read<0>();  // staged tiles must be read out before shared memory goes away
    }
    __syncthreads();
    if (threadIdx.x == 0) trace_mark(a.trace, 3);
}

// ============================================================================ normal mode, wide tiles
// One 128 (tokens) x 256 (weight rows) tile per CTA at a time.  Consumer warpgroup cw owns token rows [64 cw, 64 cw + 64)
// and all 256 columns: one m64n256k16 per k16 step, 128 fp32 accumulators per thread, and both consumers read the same
// weight slice, so a k-block moves 48 KB through the ring where two 128 x 128 tiles move 64 KB.  SwiGLU: the 256 weight
// rows are 128 gate rows then the 128 up rows of the same features, a tile writes 128 output features, and each thread
// holds gate (acc[i]) and up (acc[i + 64]) of its outputs.  The two consumers finish a tile together, so the epilogue is
// not hidden behind a main loop; the producer runs ahead into the next tile meanwhile.  Staging: the whole 64 x 256
// quarter of each consumer (4 slabs of [64 rows x 64 columns]); a plain residual is TMA-loaded into it during the main loop.
template <int STAGES, int EPI>
__global__ void __launch_bounds__(TOK_THREADS, 1)
gemm_tok_wide_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                     const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_res, const GemmArgs a) {
    static_assert(EPI >= 0 && !(EPI & EPI_F32OUT), "compile-time epilogue with a TMA store");
    using Cfg = WideCfg<STAGES>;
    extern __shared__ uint8_t smem_raw[];
    const TokSmem<Cfg> sm(smem_raw);

    const int wg = threadIdx.x >> 7;
    const int tw = threadIdx.x & 127;
    constexpr int flags = EPI;
    constexpr bool swiglu = flags & EPI_SWIGLU;
    constexpr int OUT_COLS = swiglu ? 128 : 256;  // output columns of a tile
    constexpr bool tma_res = flags & EPI_RESID;  // plain residual only (the host keeps periodic ones on the 128 x 128 kernel)

    // `empty`: 8 arrivals, one per consumer warp, since both warpgroups read every stage; no `order` barriers
    if (threadIdx.x == 0) tok_prologue(sm, 8, false, a, &map_x, &map_w, &map_out, &map_res, true, tma_res);
    __syncthreads();
    pdl_launch_dependents();  // the next kernel may start its prologue behind us

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (tw == 0) {
            pdl_wait();
            tok_produce(sm, &map_x, a, [&](uint8_t* sW, uint64_t* bar, int k0, int c) {
                // the two 128-row halves: plain, or one 256-row block of the gate / up interleaved layout, or gate and up of [gate; up]
                const bool concat = swiglu && a.swiglu_up_row0;
                tma_load_2d(sW, &map_w, bar, k0, concat ? c * 128 : c * 256);
                tma_load_2d(sW + Cfg::W_BYTES / 2, &map_w, bar, k0, concat ? a.swiglu_up_row0 + c * 128 : c * 256 + 128);
            });
        }
    } else {
        setmaxnreg_inc<232>();
        const int cw = wg - 1;  // consumer index: token rows [64 cw, 64 cw + 64) of the tile
        const bool leader = tw == 0;
        const typename Cfg::Out slabs{sm.staging + cw * Cfg::Out::BYTES};
        const int num_tiles = a.num_r_tiles * a.num_c_tiles;
        const int kb_n = (a.K + BK - 1) / BK;
        pdl_wait();  // residual reads / output writes are ordered after every earlier kernel
        if (threadIdx.x == 128) trace_mark(a.trace, 1);
        uint32_t rpar = 0;
        Ring<STAGES> ring;
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            int r, c;
            tile_coords(t, a, r, c);
            const int row0 = r * 128 + cw * 64;  // first token row of this warpgroup
            const int out_col0 = c * OUT_COLS;
            // residual slabs of this tile: they arrive while the main loop runs
            if (tma_res && leader) slabs.load_res(&map_res, &sm.rbar[cw], out_col0, row0, a.n_feat);

            // ---- main loop: one m64n256k16 per k16 step
            float acc[128];
#pragma unroll
            for (int i = 0; i < 128; ++i) acc[i] = 0.f;
            auto fence = [&] { fence_regs(acc); };
            const int held = ring_mma(ring, sm.full, sm.empty, kb_n, [&](int stage) {
                const uint32_t sX = smem_u32(sm.ring + stage * Cfg::STAGE_BYTES) + cw * 64 * 128;
                const uint32_t sW = smem_u32(sm.ring + stage * Cfg::STAGE_BYTES) + Cfg::X_BYTES;
#pragma unroll
                for (int k = 0; k < BK / 16; ++k)
                    wgmma_m64n256_ss<0, 0>(acc, make_smem_desc_sw128(sX + k * 32, 0, 1024), make_smem_desc_sw128(sW + k * 32, 0, 1024), 1);
            }, fence);
            ring_drain(sm.empty, held, fence);
            if (threadIdx.x == 128) trace_mark(a.trace, 2);

            // ---- epilogue from the accumulator fragments
            slabs.acquire(leader, tma_res, 1 + cw, &sm.rbar[cw], rpar);
            epi_fragment<256, tma_res ? 1 : 0>(acc, slabs, 0, row0, out_col0, flags, a);
            slabs.store(leader, 1 + cw, &map_out, OUT_COLS / 64, out_col0, row0, a.n_feat);
        }
        if (leader) bulk_wait_read<0>();  // staged tiles must be read out before shared memory goes away
    }
    __syncthreads();
    if (threadIdx.x == 0) trace_mark(a.trace, 3);
}

// ============================================================================ normal mode, FP8 (gemm_fp8, n_tok > 64)
// One 128 (tokens) x 128 (weight rows) tile per CTA at a time, both operands block-scaled e4m3.  Consumer warpgroup cw owns
// token rows [64 cw, 64 cw + 64) and all 128 columns: four m64n128k32 QGMMAs per k-block into a k-block accumulator (64
// fp32), which is then promoted into the main accumulator (64 fp32) with sx of the thread's two token rows times sw of the
// column's 128-row weight block.  A 128 x 128 tile per warpgroup would need 256 accumulator registers per thread.  The weight
// rows of a tile are two 64-row halves: rows [128 c, 128 c + 128), or with SwiGLU the 64 gate rows 64 c.. and the 64 up rows
// of the same features of the [gate; up] layout, which lie in different scale blocks -- hence one scale per column half.
// The epilogue rounds the result to bf16 (FP8Linear's output) and then runs the bf16 kernels' register epilogue.
template <int STAGES, int EPI>
__global__ void __launch_bounds__(TOK_THREADS, 1)
gemm_fp8_tok_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                    const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_res, const GemmArgs a) {
    static_assert(EPI >= 0 && !(EPI & (EPI_F32OUT | EPI_GELU | EPI_ROPE)), "FP8 epilogues: bias, residual, SwiGLU");
    using Cfg = Fp8TokCfg<STAGES>;
    extern __shared__ uint8_t smem_raw[];
    const TokSmem<Cfg> sm(smem_raw);

    const int wg = threadIdx.x >> 7;
    const int tw = threadIdx.x & 127;
    constexpr int flags = EPI;
    constexpr bool swiglu = flags & EPI_SWIGLU;
    constexpr int OUT_COLS = swiglu ? 64 : 128;
    constexpr bool tma_res = flags & EPI_RESID;

    // `empty`: 8 arrivals, one per consumer warp, since both warpgroups read every stage
    if (threadIdx.x == 0) tok_prologue(sm, 8, false, a, &map_x, &map_w, &map_out, &map_res, true, tma_res);
    __syncthreads();
    pdl_launch_dependents();

    // weight-row halves of column tile c
    auto w_row = [&](int c, int h) { return swiglu ? h * a.swiglu_up_row0 + c * 64 : c * 128 + h * 64; };
    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (tw == 0) {
            pdl_wait();
            tok_produce(sm, &map_x, a, [&](uint8_t* sW, uint64_t* bar, int k0, int c) {
                tma_load_2d(sW, &map_w, bar, k0, w_row(c, 0));
                tma_load_2d(sW + 64 * 128, &map_w, bar, k0, w_row(c, 1));
            });
        }
    } else {
        setmaxnreg_inc<232>();
        const int cw = wg - 1;
        const bool leader = tw == 0;
        const typename Cfg::Out slabs{sm.staging + cw * Cfg::Out::BYTES};
        const int num_tiles = a.num_r_tiles * a.num_c_tiles;
        const int kb_n = a.K / 128;
        pdl_wait();  // activation scales, residual reads and output writes are ordered after every earlier kernel
        if (threadIdx.x == 128) trace_mark(a.trace, 1);
        uint32_t rpar = 0;
        Ring<STAGES> ring;
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            int r, c;
            tile_coords(t, a, r, c);
            const int row0 = r * 128 + cw * 64;
            const int out_col0 = c * OUT_COLS;
            if (tma_res && leader) slabs.load_res(&map_res, &sm.rbar[cw], out_col0, row0, a.n_feat);
            // scale rows: sw of the two column halves, sx of this thread's two token rows (0 past n_tok)
            const float* swp0 = a.sw + static_cast<size_t>(w_row(c, 0) / 128) * a.ld_sw;
            const float* swp1 = a.sw + static_cast<size_t>(w_row(c, 1) / 128) * a.ld_sw;
            const int tok0 = row0 + frag_row(tw, 0), tok1 = row0 + frag_row(tw, 2);
            const bool ok0 = tok0 < a.n_tok, ok1 = tok1 < a.n_tok;

            float acc[64], kacc[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = kacc[i] = 0.f;
            for (int kb = 0; kb < kb_n; ++kb) {
                const float sw0 = __ldg(swp0 + kb), sw1 = __ldg(swp1 + kb);
                const float sx0 = ok0 ? a.sx[static_cast<size_t>(kb) * a.n_tok + tok0] : 0.f;
                const float sx1 = ok1 ? a.sx[static_cast<size_t>(kb) * a.n_tok + tok1] : 0.f;
                mbar_wait(&sm.full[ring.stage], ring.phase);
                const uint32_t sX = smem_u32(sm.ring + ring.stage * Cfg::STAGE_BYTES) + cw * 64 * 128;
                const uint32_t sW = smem_u32(sm.ring + ring.stage * Cfg::STAGE_BYTES) + Cfg::X_BYTES;
                fence_regs(kacc);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    wgmma_m64n128k32_e4m3(kacc, make_smem_desc_sw128(sX + k * 32, 0, 1024), make_smem_desc_sw128(sW + k * 32, 0, 1024), k > 0);
                wgmma_commit();
                wgmma_wait<0>();  // the k-block's partial sums are final: promote them
                fence_regs(kacc);
                if ((tw & 31) == 0) mbar_arrive(&sm.empty[ring.stage]);
                ring.next();
                const float s00 = sx0 * sw0, s01 = sx0 * sw1, s10 = sx1 * sw0, s11 = sx1 * sw1;
#pragma unroll
                for (int i = 0; i < 64; ++i) {
                    // register i: row +8 when (i >> 1) & 1, column 8 (i >> 2) + ...: the upper column half from i = 32 on
                    const float sc = ((i >> 1) & 1) ? (i < 32 ? s10 : s11) : (i < 32 ? s00 : s01);
                    acc[i] = fmaf(kacc[i], sc, acc[i]);
                }
            }
            if (threadIdx.x == 128) trace_mark(a.trace, 2);
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = bf16_round(acc[i]);  // FP8Linear returns its matmul in bf16

            slabs.acquire(leader, tma_res, 1 + cw, &sm.rbar[cw], rpar);
            epi_fragment<128, tma_res ? 1 : 0>(acc, slabs, 0, row0, out_col0, flags, a);
            slabs.store(leader, 1 + cw, &map_out, OUT_COLS / 64, out_col0, row0, a.n_feat);
        }
        if (leader) bulk_wait_read<0>();
    }
    __syncthreads();
    if (threadIdx.x == 0) trace_mark(a.trace, 3);
}

// ============================================================================ few-token (swap) mode (n_tok <= 64)
// EPI >= 0: epilogue flags fixed at compile time (no per-element branches, full ILP across the 32-column chunk);
// EPI < 0: generic instantiation reading a.flags at run time (odd layouts / unusual flag mixes).
// FP8: both operands e4m3 with block scales (gemm_fp8).  A stage then holds 128 K (one 128-byte swizzle row = one scale
// group) in the same bytes as 64 bf16 K.  Each k-block is accumulated by m64n32k32 QGMMAs into its own registers and
// promoted into the fp32 accumulator with sw (of the weight rows' 128-row block) x sx (of each token column), so the
// tensor-core accumulation never spans two k-blocks.  The epilogue first rounds the result to bf16 (FP8Linear's output).
template <int BN, int NA, int STAGES, int EPI, bool FP8 = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap map_r, const __grid_constant__ CUtensorMap map_c, const GemmArgs a) {
    using Cfg = GemmCfg<BN, NA, STAGES>;
    constexpr int KB = FP8 ? 128 : BK;  // K elements per k-block (128 bytes of every row either way)
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    float* accbuf = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint8_t* epi_stage = smem + STAGES * Cfg::STAGE_BYTES + Cfg::ACC_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(epi_stage + Cfg::EPI_STAGE_BYTES);
    uint64_t* empty = full + STAGES;
    uint32_t* flag_slot = reinterpret_cast<uint32_t*>(empty + STAGES);

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
        fence_barrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();  // the next kernel may start its prologue / weight prefetch behind us

    const int k_splits = a.k_splits;
    const int num_tiles = a.num_r_tiles * a.num_c_tiles * k_splits;  // work items: (tile, split), split fastest
    const int k_blocks_total = (a.K + KB - 1) / KB;
    // K range of split s: blocks [kb_lo(s), kb_lo(s+1)), sizes differ by at most one
    auto kb_lo = [&](int s) { return (s * k_blocks_total) / k_splits; };

    if (warp == 8) {
        if constexpr (FP8) {
            // the weight scales of the first work item, like its weights, do not depend on earlier kernels: into L2 now
            if (blockIdx.x < num_tiles) {
                int r, c;
                tile_coords(blockIdx.x / k_splits, a, r, c);
#pragma unroll
                for (int na = 0; na < NA; ++na) {
                    const float* row = a.sw + static_cast<size_t>(a.swiglu_up_row0 ? (na * a.swiglu_up_row0) / 128 + r : r * NA + na) * a.ld_sw;
                    for (int j = lane * 32; j < a.ld_sw; j += 32 * 32) prefetch_l2(row + j);
                }
            }
        }
        if (lane == 0) {
            Ring<STAGES> ring;
            // The row operand is a WEIGHT matrix, independent of earlier kernels -> its first STAGES tiles are
            // requested before pdl_wait(), so weight streaming overlaps the tail of the previous kernel(s).
            int prefetched = 0;
            {
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
                            tma_load_2d(sR + na * 128 * BK * 2, &map_r, &full[prefetched], kb * KB,
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
                    uint8_t* sR = smem + ring.stage * Cfg::STAGE_BYTES;
                    uint8_t* sC = sR + Cfg::R_BYTES;
                    if (issued >= prefetched) {
                        mbar_wait(&empty[ring.stage], ring.phase ^ 1);
                        mbar_arrive_expect_tx(&full[ring.stage], Cfg::STAGE_BYTES);
#pragma unroll
                        for (int na = 0; na < NA; ++na)
                            tma_load_2d(sR + na * 128 * BK * 2, &map_r, &full[ring.stage], kb * KB,
                                        a.swiglu_up_row0 ? na * a.swiglu_up_row0 + r * 128 : (r * NA + na) * 128);
                    }
                    tma_load_2d(sC, &map_c, &full[ring.stage], kb * KB, c * BN);
                    ring.next();
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
        const int row_in_tile = q * 32 + lane;
        const bool epi_warp = warp < 4;
        pdl_wait();  // residual reads / output writes / split-K workspace are ordered after every earlier kernel
        if (threadIdx.x == 0) trace_mark(a.trace, 1);
        Ring<STAGES> ring;
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            {
                const int sp = t % k_splits;
                float accr[NA][BN / 2];
#pragma unroll
                for (int na = 0; na < NA; ++na)
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) accr[na][i] = 0.f;
                auto fence = [&] {
#pragma unroll
                    for (int na = 0; na < NA; ++na) fence_regs(accr[na]);
                };
                if constexpr (FP8) {
                    int r, c;
                    tile_coords(t / k_splits, a, r, c);
                    // sw rows of the NA 128-row weight blocks; sx of this thread's 8 token columns (frag_col), 0 past n_tok
                    const float* swp[NA];
#pragma unroll
                    for (int na = 0; na < NA; ++na)
                        swp[na] = a.sw + static_cast<size_t>(a.swiglu_up_row0 ? (na * a.swiglu_up_row0) / 128 + r : r * NA + na) * a.ld_sw;
                    const float* sxp[8];
                    bool sx_ok[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int tok = c * BN + frag_col(tw, 2 * (j >> 1) * 2 + (j & 1));
                        sx_ok[j] = tok < a.n_tok;
                        sxp[j] = a.sx + (sx_ok[j] ? tok : 0);
                    }
                    float kacc[NA][BN / 2];
#pragma unroll
                    for (int na = 0; na < NA; ++na)
#pragma unroll
                        for (int i = 0; i < BN / 2; ++i) kacc[na][i] = 0.f;
                    const bool lane0 = lane == 0;
                    for (int kb = kb_lo(sp); kb < kb_lo(sp + 1); ++kb) {
                        // scales first: their loads are in flight while the stage lands
                        float sw[NA], sx[8];
#pragma unroll
                        for (int na = 0; na < NA; ++na) sw[na] = __ldg(swp[na] + kb);
#pragma unroll
                        for (int j = 0; j < 8; ++j) sx[j] = sx_ok[j] ? sxp[j][static_cast<size_t>(kb) * a.n_tok] : 0.f;
                        mbar_wait(&full[ring.stage], ring.phase);
                        const uint32_t sR = smem_u32(smem + ring.stage * Cfg::STAGE_BYTES);
                        const uint32_t sC = sR + Cfg::R_BYTES;
#pragma unroll
                        for (int na = 0; na < NA; ++na) fence_regs(kacc[na]);
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const uint64_t bdesc = make_smem_desc_sw128(sC + k * 32, 0, 1024);
#pragma unroll
                            for (int na = 0; na < NA; ++na) {
                                const uint64_t adesc = make_smem_desc_sw128(sR + na * 128 * BK * 2 + wg * 64 * 128 + k * 32, 0, 1024);
                                wgmma_m64n32k32_e4m3(kacc[na], adesc, bdesc, k > 0);
                            }
                        }
                        wgmma_commit();
                        wgmma_wait<0>();  // the k-block's partial sums are final: promote them
#pragma unroll
                        for (int na = 0; na < NA; ++na) fence_regs(kacc[na]);
                        if (lane0) mbar_arrive(&empty[ring.stage]);
                        ring.next();
#pragma unroll
                        for (int na = 0; na < NA; ++na)
#pragma unroll
                            for (int i = 0; i < BN / 2; ++i) {
                                // register i holds column frag_col(tw, i): column pair (i >> 2, i & 1) of this thread
                                const int j = 2 * (i >> 2) + (i & 1);
                                accr[na][i] = fmaf(kacc[na][i], sw[na] * sx[j], accr[na][i]);
                            }
                    }
                } else {
                    const int held = ring_mma(ring, full, empty, kb_lo(sp + 1) - kb_lo(sp), [&](int stage) {
                        const uint32_t sR = smem_u32(smem + stage * Cfg::STAGE_BYTES);
                        const uint32_t sC = sR + Cfg::R_BYTES;
#pragma unroll
                        for (int k = 0; k < BK / 16; ++k) {
                            const uint64_t bdesc = make_smem_desc_sw128(sC + k * 32, 0, 1024);
#pragma unroll
                            for (int na = 0; na < NA; ++na) {
                                const uint64_t adesc = make_smem_desc_sw128(sR + na * 128 * BK * 2 + wg * 64 * 128 + k * 32, 0, 1024);
                                wgmma_m64n32_ss<0, 0>(accr[na], adesc, bdesc, 1);
                            }
                        }
                    }, fence);
                    ring_drain(empty, held, fence);
                }
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
            // few-token mode with a fused residual: this thread's residual vectors of the transposed epilogue (token et / 4,
            // features (et % 4) * 32 ...) do not depend on this GEMM -- request them now, they arrive while the weights stream
            // (the epilogue otherwise exposes one more L2 round trip in the split-K tail)
            [[maybe_unused]] uint4 rv_pre[4];
            [[maybe_unused]] bool rv_ok = false;
            if constexpr (NA == 1) {
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

            {
                // swapped: accumulator row = output feature, column = token
                const int feat = r * 128 + row_in_tile;
                const bool feat_ok = feat < a.n_feat;
                const float bias = ((flags & EPI_BIAS) && feat_ok) ? __bfloat162float(a.bias[feat]) : 0.f;
                uint32_t v[32], u[32];
                acc_ld32<Cfg::ACC_COLS>(accbuf, row_in_tile, 0, v);
                if constexpr (NA == 2) acc_ld32<Cfg::ACC_COLS>(accbuf, row_in_tile, BN, u);
                if constexpr (NA == 1) {
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
                if constexpr (FP8) {  // FP8Linear returns its matmul in bf16; bias / residual / SwiGLU act on that
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        v[j] = __float_as_uint(bf16_round(__uint_as_float(v[j])));
                        if constexpr (NA == 2) u[j] = __float_as_uint(bf16_round(__uint_as_float(u[j])));
                    }
                }
                const int tok0 = c * BN;
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
                                if (rv_ok) {   // requested before the accumulator wait (same token / features)
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

    __syncthreads();
    if (threadIdx.x == 0) trace_mark(a.trace, 3);
}

// One persistent CTA per SM, fewer when there are fewer work items (tiles x K splits).  The shared-memory opt-in is per
// kernel instantiation and per device, hence one DeviceOnce per kernel.
template <auto kern, int SMEM_BYTES, int THREADS, class... Maps>
static int launch_gemm(const GemmArgs& a, cudaStream_t stream, const Maps&... maps) {
    static DeviceOnce once;
    if (once.first()) {
        AF3_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    }
    const int items = a.num_r_tiles * a.num_c_tiles * a.k_splits;
    const int grid = items < sm_count() ? items : sm_count();
    AF3_CHECK_CUDA(launch_kernel(kern, dim3(grid), dim3(THREADS), SMEM_BYTES, stream, maps..., a));
    return 0;
}

template <int BN, int NA, int STAGES>
static int launch_swap(const CUtensorMap& mr, const CUtensorMap& mc, const GemmArgs& a, cudaStream_t stream) {
#define AF3_EPI_CASE(F) \
    case (F):           \
        return launch_gemm<gemm_kernel<BN, NA, STAGES, (F)>, GemmCfg<BN, NA, STAGES>::SMEM_BYTES, GEMM_THREADS>(a, stream, mr, mc);
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
#undef AF3_EPI_CASE
    return launch_gemm<gemm_kernel<BN, NA, STAGES, -1>, GemmCfg<BN, NA, STAGES>::SMEM_BYTES, GEMM_THREADS>(a, stream, mr, mc);
}

size_t gemm_workspace_bytes() { return (8u << 20) + 4096 * sizeof(int); }

// split-K of the few-token mode: when the tile grid cannot fill the GPU and a (zero-initialised) workspace was supplied,
// split the kb_total k-blocks of every tile over s CTAs
static void choose_k_splits(GemmArgs& a, int kb_total, void* workspace, size_t workspace_bytes) {
    a.k_splits = 1;
    const int tiles = a.num_r_tiles * a.num_c_tiles;
    if (workspace && workspace_bytes >= gemm_workspace_bytes() && tiles * 2 <= sm_count() && tiles <= 4096) {
        int s = sm_count() / tiles;
        const int forced = [] { const char* e = getenv("AF3_KSPLIT"); return e ? atoi(e) : 0; }();  // experiments only (read per call)
        if (forced > 0) s = forced;
        if (s > kb_total / 4) s = kb_total / 4;  // keep at least 4 k-blocks per split
        if (s > 16) s = 16;
        if (s >= 2 && static_cast<size_t>(tiles) * s * 32 * 128 * sizeof(float) <= (8u << 20)) {
            a.k_splits = s;
            a.ws = reinterpret_cast<float*>(workspace);
            a.counters = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(workspace) + (8u << 20));
        }
    }
}

// Host entry.  x: [n_tok, K] bf16 (pitch ldx), w: [n_rows_w, K] bf16 (pitch ldw) where n_rows_w = n_feat, or the
// gate/up-interleaved 2*ceil(n_feat/128)*128 rows when EPI_SWIGLU.  out: [n_tok, n_feat] (pitch ldo).
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
        a.num_r_tiles = ceil_div(n_tok, 128);
        // rasterisation: GROUP_R row tiles stay L2-resident (~20 MB of the 50 MB L2) while the col-operand tiles stream
        // past them, so the streamed operand is re-read num_r_tiles / GROUP_R times instead of once per row tile
        {
            const long long tile_bytes = 128ll * K * 2;
            long long g = (20ll << 20) / tile_bytes;
            a.group_r = static_cast<int>(g < 8 ? 8 : (g > 256 ? 256 : g));
        }
        // smem-staged TMA-store epilogue whenever the output (and residual) layout allows 16-byte-aligned rows
        const bool res_plain = (flags & EPI_RESID) && res_period == 0;
        a.tma_epi = !(flags & EPI_F32OUT) && (ldo % 8 == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0) &&
                    (!res_plain || ((ld_res % 8 == 0) && ((reinterpret_cast<uintptr_t>(resid) & 15) == 0)));
        auto launch = [&](auto epi) {
            constexpr int EPI = decltype(epi)::value;
            // 128 x 256 tiles where the main loop is long enough to pay for an epilogue that no main loop hides.  On an H100
            // 80GB HBM3 (700 W) they ran every K >= 3584 GEMM of config 2 7-15 % faster than the ping-pong kernel, but conv2
            // (K = 3840, periodic residual read from global memory in the epilogue) 8 % slower, and lost up to 10 % at K = 1280
            // (profiles/microbench_prefill_gemm.py)
            const bool wide = EPI >= 0 && K >= 2048 && res_period == 0;
            a.num_c_tiles = ceil_div(w_rows, wide ? 256 : 128);
            if (int e = make_tmap_2d(&mx, x, K, n_tok, ldx, BK, 128)) return e;
            // weight box: a 128-row half of a wide tile, a 128 x 128 tile, or the 64 gate / 64 up rows of a SwiGLU tile
            if (int e = make_tmap_2d(&mw, w, K, w_rows, ldw, BK, (swiglu && !wide) ? 64 : 128)) return e;
            mo = mx;
            mres = mx;
            if (a.tma_epi) {
                // [rows x 64 columns] slabs of a consumer warpgroup: one TMA store (residual: load) per 64 output columns
                const int slab_rows = wide ? 64 : 128;
                if (int e = make_tmap_2d(&mo, out, n_feat, n_tok, ldo, 64, slab_rows)) return e;
                if (res_plain)
                    if (int e = make_tmap_2d(&mres, resid, n_feat, n_tok, ld_res, 64, slab_rows)) return e;
            }
            if constexpr (EPI >= 0)
                if (wide)
                    return launch_gemm<gemm_tok_wide_kernel<WIDE_STAGES, EPI>, WideCfg<WIDE_STAGES>::SMEM_BYTES, TOK_THREADS>(
                        a, stream, mx, mw, mo, mres);
            return launch_gemm<gemm_tok_kernel<TOK_STAGES, EPI>, TokCfg<TOK_STAGES>::SMEM_BYTES, TOK_THREADS>(a, stream, mx, mw,
                                                                                                              mo, mres);
        };
        // compile-time epilogues for the flag sets the AF3 path uses, only with the TMA-store epilogue; anything else runs the
        // generic instantiation (128 x 128 tiles)
        if (a.tma_epi) {
            switch (flags) {
#define AF3_EPI_CASE(F) \
    case (F):           \
        return launch(IntC<(F)>{});
                AF3_EPI_CASE(0)
                AF3_EPI_CASE(EPI_BIAS)
                AF3_EPI_CASE(EPI_BIAS | EPI_GELU)
                AF3_EPI_CASE(EPI_BIAS | EPI_RESID)
                AF3_EPI_CASE(EPI_RESID)
                AF3_EPI_CASE(EPI_SWIGLU)
                AF3_EPI_CASE(EPI_BIAS | EPI_GELU | EPI_RESID)
#undef AF3_EPI_CASE
                default:
                    break;
            }
        }
        return launch(IntC<-1>{});
    }
    constexpr int BN = 32;
    a.num_c_tiles = ceil_div(n_tok, BN);
    a.group_r = 1;
    if (int e = make_tmap_2d(&mw, w, K, w_rows, ldw, BK, 128)) return e;
    if (int e = make_tmap_2d(&mx, x, K, n_tok, ldx, BK, BN)) return e;
    // Pipeline depth of the few-token mode: 10 x 20 KB (NA = 1) / 5 x 36 KB (NA = 2) stages, as deep as the 227 KB of shared memory
    // allows next to the accumulator tile: the weight streams of a few-token GEMM are latency-bound on the bytes in flight per SM.
    if (swiglu) {
        a.num_r_tiles = ceil_div(w_rows, 256);
        return launch_swap<BN, 2, 5>(mw, mx, a, stream);
    }
    a.num_r_tiles = ceil_div(w_rows, 128);
    choose_k_splits(a, ceil_div(K, BK), workspace, workspace_bytes);
    // ring depth: 10 x 20 KB = 200 KB in flight per SM (the few-token streams are latency-bound on bytes in flight)
    return launch_swap<BN, 1, 10>(mw, mx, a, stream);
}

// Host entry of the block-scaled FP8 GEMM (include/af3b200.h af3_gemm_fp8): up to 64 tokens the few-token kernel with e4m3
// operands (split-K, RoPE epilogue), above that gemm_fp8_tok_kernel.  Epilogues: none, bias, residual, SwiGLU on [gate; up],
// bias + RoPE + KV append (few-token only).
int gemm_fp8(cudaStream_t stream, const uint8_t* x, int ldx, const float* sx, const uint8_t* w, int ldw, const float* sw,
             void* out, int ldo, int n_tok, int n_feat, int K, int flags, const bf16* bias, const bf16* resid, int ld_res,
             void* workspace, size_t workspace_bytes, const RopeEpilogue* rope) {
    AF3_REQUIRE(n_tok > 0 && n_feat > 0 && K > 0, "gemm_fp8: empty problem");
    AF3_REQUIRE(K % 128 == 0 && n_feat % 128 == 0, "gemm_fp8: K and n_feat must be multiples of 128 (the scale blocks)");
    AF3_REQUIRE(ldx % 16 == 0 && ldw % 16 == 0 && ldx >= K && ldw >= K, "gemm_fp8: pitches must be multiples of 16 bytes");
    AF3_REQUIRE(sx && sw, "gemm_fp8: scale pointers required");
    AF3_REQUIRE(!(flags & EPI_BIAS) || bias, "gemm_fp8: bias flag without pointer");
    AF3_REQUIRE(!(flags & EPI_RESID) || resid, "gemm_fp8: residual flag without pointer");
    const bool swiglu = flags & EPI_SWIGLU;
    AF3_REQUIRE(!swiglu || (flags & EPI_SWIGLU_CONCAT), "gemm_fp8: SwiGLU needs the [gate; up] layout (AF3_EPI_SWIGLU_CONCAT)");
    flags &= ~EPI_SWIGLU_CONCAT;
    const bool rope_epi = flags & EPI_ROPE;
    AF3_REQUIRE(flags == 0 || flags == EPI_BIAS || flags == EPI_RESID || flags == EPI_SWIGLU || flags == (EPI_BIAS | EPI_ROPE),
                "gemm_fp8: supported epilogues are none, bias, residual, SwiGLU and bias + RoPE");
    AF3_REQUIRE((ldo % 8) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0, "gemm_fp8: out must be 16-byte aligned, ldo % 8 == 0");
    AF3_REQUIRE(!(flags & EPI_RESID) || ((ld_res % 8) == 0 && (reinterpret_cast<uintptr_t>(resid) & 15) == 0),
                "gemm_fp8: resid must be 16-byte aligned, ld_res % 8 == 0");
    const int w_rows = swiglu ? 2 * n_feat : n_feat;
    GemmArgs a{};
    a.K = K;
    a.n_tok = n_tok;
    a.n_feat = n_feat;
    a.out = out;
    a.ldo = ldo;
    a.bias = bias;
    a.resid = resid;
    a.ld_res = ld_res;
    a.flags = flags;
    a.swiglu_up_row0 = swiglu ? n_feat : 0;
    a.sx = sx;
    a.sw = sw;
    a.ld_sw = K / 128;
    a.k_splits = 1;
    a.trace = trace_next_slot();
    if (rope_epi) {
        AF3_REQUIRE(rope && rope->cs && rope->k_cache && rope->v_cache && rope->pos, "gemm_fp8: EPI_ROPE needs the rope arguments");
        AF3_REQUIRE(n_tok <= 64 && n_feat == (rope->H + 2 * rope->Hkv) * 128, "gemm_fp8: EPI_ROPE is the few-token fused q/k/v projection with head_dim 128");
        a.rope_cs = reinterpret_cast<const float2*>(rope->cs);
        a.k_cache = rope->k_cache;
        a.v_cache = rope->v_cache;
        a.rope_pos = rope->pos;
        a.rope_H = rope->H;
        a.rope_Hkv = rope->Hkv;
        a.rope_Tmax = rope->Tmax;
    }
    if (n_tok > 64) {
        // token-major tiles: rows = tokens, cols = 128 weight rows (64 outputs with SwiGLU)
        a.num_r_tiles = ceil_div(n_tok, 128);
        a.num_c_tiles = w_rows / 128;
        {  // as gemm_bf16: GROUP_R token tiles (~20 MB) stay L2-resident while the weight tiles stream past them
            const long long g = (20ll << 20) / (128ll * K);
            a.group_r = static_cast<int>(g < 8 ? 8 : (g > 256 ? 256 : g));
        }
        CUtensorMap mx, mw, mo, mres;
        if (int e = make_tmap_2d_u8(&mx, x, K, n_tok, ldx, 128, 128)) return e;
        if (int e = make_tmap_2d_u8(&mw, w, K, w_rows, ldw, 128, 64)) return e;
        if (int e = make_tmap_2d(&mo, out, n_feat, n_tok, ldo, 64, 64)) return e;
        mres = mo;
        if (flags & EPI_RESID)
            if (int e = make_tmap_2d(&mres, resid, n_feat, n_tok, ld_res, 64, 64)) return e;
        switch (flags) {
#define AF3_EPI_CASE(F) \
    case (F):           \
        return launch_gemm<gemm_fp8_tok_kernel<FP8_TOK_STAGES, (F)>, Fp8TokCfg<FP8_TOK_STAGES>::SMEM_BYTES, TOK_THREADS>(a, stream, mx, mw, mo, mres);
            AF3_EPI_CASE(0)
            AF3_EPI_CASE(EPI_BIAS)
            AF3_EPI_CASE(EPI_RESID)
            AF3_EPI_CASE(EPI_SWIGLU)
#undef AF3_EPI_CASE
            default:
                return fail("gemm_fp8: unsupported epilogue");
        }
    }
    constexpr int BN = 32;
    a.num_c_tiles = ceil_div(n_tok, BN);
    a.num_r_tiles = ceil_div(w_rows, swiglu ? 256 : 128);
    a.group_r = 1;
    CUtensorMap mw, mx;
    if (int e = make_tmap_2d_u8(&mw, w, K, w_rows, ldw, 128, 128)) return e;
    if (int e = make_tmap_2d_u8(&mx, x, K, n_tok, ldx, 128, BN)) return e;
    if (swiglu)  // ring depth as in gemm_bf16: as many stages as fit beside the accumulator tile
        return launch_gemm<gemm_kernel<BN, 2, 5, EPI_SWIGLU, true>, GemmCfg<BN, 2, 5>::SMEM_BYTES, GEMM_THREADS>(a, stream, mw, mx);
    choose_k_splits(a, K / 128, workspace, workspace_bytes);
    switch (flags) {
#define AF3_EPI_CASE(F) \
    case (F):           \
        return launch_gemm<gemm_kernel<BN, 1, 10, (F), true>, GemmCfg<BN, 1, 10>::SMEM_BYTES, GEMM_THREADS>(a, stream, mw, mx);
        AF3_EPI_CASE(0)
        AF3_EPI_CASE(EPI_BIAS)
        AF3_EPI_CASE(EPI_RESID)
        AF3_EPI_CASE(EPI_BIAS | EPI_ROPE)
#undef AF3_EPI_CASE
        default:
            return fail("gemm_fp8: unsupported epilogue");
    }
}

// ============================================================================ LM head + cross-entropy (lm_head_xent)
// A label is counted when it lies in [0, V) and is not ignore_index; one outside [0, V) that is not ignore_index is invalid:
// never used as an index, counted as ignored and reported in totals[2].
__device__ __forceinline__ bool xent_counted(long long lab, int V, long long ignore_index) { return lab >= 0 && lab < V && lab != ignore_index; }

// One warp per token: lse from the token's column-tile partials, merged in a fixed order (lane j takes tiles j, j + 32, ...
// in order, then a butterfly across the warp), and nll = lse - logit[label], 0 for an uncounted position.
__global__ void __launch_bounds__(256)
xent_merge_kernel(const float2* __restrict__ part, const float* __restrict__ tgt, const int64_t* __restrict__ labels, int n_tok,
                  int n_ct, int V, long long ignore_index, float* __restrict__ token_nll) {
    const int tok = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (tok >= n_tok) return;
    if (!xent_counted(labels[tok], V, ignore_index)) {
        if (lane == 0) token_nll[tok] = 0.f;
        return;
    }
    const float2* p = part + static_cast<size_t>(tok) * n_ct;
    float m = -INFINITY;
    for (int j = lane; j < n_ct; j += 32) m = fmaxf(m, p[j].x);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int j = lane; j < n_ct; j += 32) {
        const float2 q = p[j];
        s += q.y * expf(q.x - m);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) token_nll[tok] = m + logf(s) - tgt[tok];
}

// One CTA: totals = {sum of nll, counted positions, invalid labels}, in fp64 and a fixed order (thread i sums tokens i,
// i + 1024, ..., then a tree over the threads).
__global__ void __launch_bounds__(1024)
xent_totals_kernel(const float* __restrict__ token_nll, const int64_t* __restrict__ labels, int n_tok, int V, long long ignore_index,
                   double* __restrict__ totals) {
    __shared__ double sh[3][1024];
    double sum = 0.0, n = 0.0, bad = 0.0;
    for (int t = threadIdx.x; t < n_tok; t += 1024) {
        const long long lab = labels[t];
        sum += token_nll[t];
        n += xent_counted(lab, V, ignore_index) ? 1.0 : 0.0;
        bad += (lab != ignore_index && (lab < 0 || lab >= V)) ? 1.0 : 0.0;
    }
    sh[0][threadIdx.x] = sum;
    sh[1][threadIdx.x] = n;
    sh[2][threadIdx.x] = bad;
    __syncthreads();
    for (int w = 512; w > 0; w >>= 1) {
        if (threadIdx.x < w)
            for (int k = 0; k < 3; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x < 3) totals[threadIdx.x] = sh[threadIdx.x][0];
}

// scratch: the partials [n_tok][ceil(V / 128)] float2, then the label logits [n_tok] float
size_t lm_head_xent_scratch_bytes(int n_tok, int V) {
    return static_cast<size_t>(n_tok) * ceil_div(V, 128) * sizeof(float2) + static_cast<size_t>(n_tok) * sizeof(float);
}

// Always the 128 x 128 ping-pong kernel, whatever n_tok: its k order is that of gemm_bf16's token-major fp32-output launch,
// so stored logits equal what af3_gemm_bf16 returns for n_tok > 64, and the statistics do not depend on whether they are stored.
int lm_head_xent(cudaStream_t stream, const bf16* x, int ldx, const bf16* w, int ldw, int n_tok, int V, int K, const int64_t* labels,
                 int64_t ignore_index, float* logits_out, int ldo, float* token_nll, double* totals, void* scratch) {
    AF3_REQUIRE(n_tok > 0 && V > 0 && K > 0, "lm_head_xent: empty problem");
    AF3_REQUIRE((K % 8) == 0 && (ldx % 8) == 0 && (ldw % 8) == 0, "lm_head_xent: K and pitches must be multiples of 8");
    AF3_REQUIRE(labels && token_nll && totals && scratch, "lm_head_xent: labels, token_nll, totals and scratch are required");
    AF3_REQUIRE(!logits_out || ldo >= V, "lm_head_xent: ldo must be at least V");
    GemmArgs a{};
    a.K = K;
    a.n_tok = n_tok;
    a.n_feat = V;
    a.out = logits_out;
    a.ldo = ldo;
    a.flags = EPI_XENT | EPI_F32OUT;
    a.k_splits = 1;
    a.trace = trace_next_slot();
    a.num_r_tiles = ceil_div(n_tok, 128);
    a.num_c_tiles = ceil_div(V, 128);
    {  // rasterisation as gemm_bf16
        const long long g = (20ll << 20) / (128ll * K * 2);
        a.group_r = static_cast<int>(g < 8 ? 8 : (g > 256 ? 256 : g));
    }
    a.labels = labels;
    a.xent_part = reinterpret_cast<float2*>(scratch);
    a.xent_tgt = reinterpret_cast<float*>(a.xent_part + static_cast<size_t>(n_tok) * a.num_c_tiles);
    CUtensorMap mx, mw;
    if (int e = make_tmap_2d(&mx, x, K, n_tok, ldx, BK, 128)) return e;
    if (int e = make_tmap_2d(&mw, w, K, V, ldw, BK, 128)) return e;
    if (int e = launch_gemm<gemm_tok_kernel<TOK_STAGES, EPI_XENT | EPI_F32OUT>, TokCfg<TOK_STAGES>::SMEM_BYTES, TOK_THREADS>(a, stream, mx, mw, mx, mx))
        return e;
    xent_merge_kernel<<<ceil_div(n_tok, 8), 256, 0, stream>>>(a.xent_part, a.xent_tgt, labels, n_tok, a.num_c_tiles, V, ignore_index, token_nll);
    AF3_CHECK_LAUNCH();
    xent_totals_kernel<<<1, 1024, 0, stream>>>(token_nll, labels, n_tok, V, ignore_index, totals);
    AF3_CHECK_LAUNCH();
    return 0;
}

}  // namespace af3
