// Fused softmax attention on wgmma tensor cores (sm_90a) for the two multi-query shapes of the AF3 path:
//   * AF-Whisper encoder self-attention: bidirectional, 20 heads x 64, 1500 frames, optional key-padding mask
//     ([O] AF3M:116-189 -> SDPA:40-104, mask from MASK:1001-1087 / AF3M:337-351)
//   * Qwen2 decoder prefill: causal GQA 28:4 x 128 with left padding / live-cache offset ([O] Q2M:206-245 -> SDPA:40-104, MASK:882)
// replacing F.scaled_dot_product_attention.  Flash-attention structure, everything in registers:
//   * one CTA = NWG consumer warpgroups of one (batch, head); warpgroup w owns 64 query rows, all of them share every K / V tile
//     (loaded once by TMA into a ring of 128-key slots, 128B-swizzled, completion on mbarriers);
//   * S = Q K^T: wgmma m64 x 128 x 16 with both operands from shared memory, fp32 in registers;
//   * online softmax on the accumulator fragment (row max / sum across the four threads of a quad), P rounded to bf16 and fed
//     back as the register A operand of O += P V (wgmma m64 x D x 16, V as the MN-major B operand straight from the row-major tile).
// Thread 0 also issues the TMA loads: a slot is refilled as soon as every warp has released it.
// Scores never touch HBM; HBM traffic is Q + K + V + O once per (batch, head) (K/V re-reads hit L2).
// NWG = 2 is the default (128 query rows per K/V tile load); NWG = 1 (AF3_ATTN_V1=1) is kept as the cross-check of the tile-range
// and masking arithmetic at a different row tiling.
#include <stdlib.h>

#include "common.h"
#include "ptx.cuh"

namespace af3 {

constexpr int AT_BN = 128;   // keys per tile
constexpr float LOG2E = 1.4426950408889634f;

// 2^x on the SFU (ex2.approx.ftz): relative error ~2^-22, far below the bf16 rounding applied to P; 2^-inf = +0
__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

struct AttnArgs {
    int Tq, Tk, H, Hkv, causal, kv_layout;
    float scale_log2;  // softmax scale * log2(e)
    const int* kv_len;
    const int* kv_start;
    bf16* out;
    int ldo;
};

template <int D, int NWG>
struct AttnCfg {
    static constexpr int BM = 64 * NWG;                    // query rows per CTA
    static constexpr int NSTG = (D == 128) ? 4 : 6;        // ring slots (one K or V tile each)
    static constexpr int TILE_BYTES = AT_BN * D * 2;
    static constexpr int Q_BYTES = BM * D * 2;
    static constexpr int SMEM_BYTES = Q_BYTES + NSTG * TILE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
    static_assert(SMEM_BYTES <= 232448, "shared memory per CTA");
};

// key tiles [j_lo, j_hi) the query rows [q0, q0 + bm) have to visit
__device__ __forceinline__ void attn_tile_range(const AttnArgs& a, int b, int q0, int bm, int& j_lo, int& j_hi) {
    const int kvl = a.kv_len ? min(a.kv_len[b], a.Tk) : a.Tk;
    const int kvs = a.kv_start ? a.kv_start[b] : 0;
    int hi_key = kvl;  // exclusive
    if (a.causal) hi_key = min(hi_key, q0 + bm - 1 + (a.Tk - a.Tq) + 1);
    j_lo = kvs / AT_BN;
    j_hi = (hi_key + AT_BN - 1) / AT_BN;
    if (j_hi < j_lo) j_hi = j_lo;
}

template <int D, int NWG>
__global__ void __launch_bounds__(128 * NWG, 1)
attention_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                 const __grid_constant__ CUtensorMap map_v, const AttnArgs a) {
    using Cfg = AttnCfg<D, NWG>;
    constexpr int DB = D / 64;        // 64-wide (128-byte) column blocks per tile
    constexpr int NSTG = Cfg::NSTG;
    constexpr int OR = D / 2;         // O accumulator registers per thread (m64 x D)
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sQ = smem;                                   // DB blocks of [BM rows][128 B]
    uint8_t* sKV = sQ + Cfg::Q_BYTES;                     // NSTG slots of DB blocks [128 keys][128 B]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + NSTG * Cfg::TILE_BYTES);
    uint64_t* q_full = bars;
    uint64_t* kv_full = bars + 1;
    uint64_t* kv_empty = kv_full + NSTG;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = warp >> 2, tw = threadIdx.x & 127;
    const int q0 = blockIdx.x * Cfg::BM, h = blockIdx.y, b = blockIdx.z;
    const int hk = h / (a.H / a.Hkv);

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&map_q);
        tma_prefetch_desc(&map_k);
        tma_prefetch_desc(&map_v);
        mbar_init(q_full, 1);
        for (int i = 0; i < NSTG; ++i) {
            mbar_init(&kv_full[i], 1);
            mbar_init(&kv_empty[i], 4 * NWG);   // one arrival per warp
        }
        fence_barrier_init();
    }
    __syncthreads();

    int j_lo, j_hi;
    attn_tile_range(a, b, q0, Cfg::BM, j_lo, j_hi);
    const int n_tiles = j_hi - j_lo;
    const int n_loads = 2 * n_tiles;  // K_t is load 2t, V_t is load 2t + 1; load i lives in slot i % NSTG

    auto issue_load = [&](int i) {   // thread 0 only
        const int slot = i % NSTG, t = i >> 1;
        mbar_arrive_expect_tx(&kv_full[slot], Cfg::TILE_BYTES);
        uint8_t* dst = sKV + slot * Cfg::TILE_BYTES;
        const CUtensorMap* mp = (i & 1) ? &map_v : &map_k;
        const int j = j_lo + t;
#pragma unroll
        for (int db = 0; db < DB; ++db) {
            if (a.kv_layout)
                tma_load_3d(dst + db * AT_BN * 128, mp, &kv_full[slot], db * 64, j * AT_BN, b * a.Hkv + hk);
            else
                tma_load_3d(dst + db * AT_BN * 128, mp, &kv_full[slot], hk * D + db * 64, j * AT_BN, b);
        }
    };
    if (threadIdx.x == 0 && n_tiles > 0) {
        mbar_arrive_expect_tx(q_full, Cfg::Q_BYTES);
#pragma unroll
        for (int db = 0; db < DB; ++db) tma_load_3d(sQ + db * Cfg::BM * 128, &map_q, q_full, h * D + db * 64, q0, b);
        for (int i = 0; i < NSTG && i < n_loads; ++i) issue_load(i);
    }
    // this thread's two query rows r0 and r0 + 8 of the fragment
    const int r0 = q0 + wg * 64 + frag_row(tw, 0);
    const int kvl = a.kv_len ? min(a.kv_len[b], a.Tk) : a.Tk;
    const int kvs = a.kv_start ? a.kv_start[b] : 0;
    const int wg_q0 = q0 + wg * 64;
    const float sl2 = a.scale_log2;
    float o[OR];
#pragma unroll
    for (int i = 0; i < OR; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    // a load's slot is free once every warp has arrived; thread 0 then refills it with load i + NSTG
    auto release = [&](int i) {
        if (lane == 0) mbar_arrive(&kv_empty[i % NSTG]);
        if (threadIdx.x == 0 && i + NSTG < n_loads) {
            mbar_wait(&kv_empty[i % NSTG], (i / NSTG) & 1);
            issue_load(i + NSTG);
        }
    };
    if (n_tiles > 0) mbar_wait(q_full, 0);
    const uint32_t aQ = smem_u32(sQ) + wg * 64 * 128;

    for (int t = 0; t < n_tiles; ++t) {
        const int k0 = (j_lo + t) * AT_BN;
        // ---- S = Q K_t^T
        float s[64];
        {
            const int i = 2 * t, slot = i % NSTG;
            mbar_wait(&kv_full[slot], (i / NSTG) & 1);
            const uint32_t aK = smem_u32(sKV + slot * Cfg::TILE_BYTES);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < D / 16; ++kk)
                wgmma_m64n128_ss<0, 0>(s, make_smem_desc_sw128(aQ + (kk >> 2) * Cfg::BM * 128 + (kk & 3) * 32, 0, 1024),
                                       make_smem_desc_sw128(aK + (kk >> 2) * AT_BN * 128 + (kk & 3) * 32, 0, 1024), kk != 0);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(s);
            release(i);
        }
        // ---- mask (only tiles that cross a boundary of some row of this warpgroup) and row maxima
        const bool need_mask = (k0 < kvs) || (k0 + AT_BN > kvl) || (a.causal && k0 + AT_BN - 1 > wg_q0 + (a.Tk - a.Tq));
        if (need_mask) {
#pragma unroll
            for (int i = 0; i < 64; ++i) {
                const int key = k0 + frag_col(tw, i);
                const int row = r0 + (((i >> 1) & 1) << 3);
                const bool ok = key >= kvs && key < kvl && (!a.causal || key <= row + (a.Tk - a.Tq));
                s[i] = ok ? s[i] : -INFINITY;
            }
        }
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 64; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
        float alpha[2], neg_m[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r] * sl2);   // sl2 > 0: max commutes with the scale
            alpha[r] = (m_run[r] == -INFINITY) ? 0.f : fast_exp2(m_run[r] - m_new);
            m_run[r] = m_new;
            neg_m[r] = (m_new == -INFINITY) ? 0.f : -m_new;
        }
        // ---- P = 2^(s * scale - m) -> bf16 A fragments; partial row sums; rescale O
        uint32_t pa[8][4];
        float ls[2] = {0.f, 0.f};
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int i = 8 * kk + 2 * e, r = e & 1;
                const float p0 = fast_exp2(fmaf(s[i], sl2, neg_m[r]));
                const float p1 = fast_exp2(fmaf(s[i + 1], sl2, neg_m[r]));
                ls[r] += p0 + p1;
                pa[kk][e] = pack_bf16x2(p0, p1);
            }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * alpha[r] + ls[r];
#pragma unroll
        for (int i = 0; i < OR; ++i) o[i] *= alpha[(i >> 1) & 1];
        // ---- O += P V_t
        {
            const int i = 2 * t + 1, slot = i % NSTG;
            mbar_wait(&kv_full[slot], (i / NSTG) & 1);
            const uint32_t aV = smem_u32(sKV + slot * Cfg::TILE_BYTES);
            fence_regs(o);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < AT_BN / 16; ++kk) {
                const uint64_t bdesc = make_smem_desc_sw128(aV + kk * 2048, AT_BN * 128, 1024);
                if constexpr (D == 128)
                    wgmma_m64n128_rs<1>(o, pa[kk], bdesc, 1);
                else
                    wgmma_m64n64_rs<1>(o, pa[kk], bdesc, 1);
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(o);
            release(i);
        }
    }

    // ---- epilogue: O / l -> bf16 -> global (the four threads of a quad hold one row's partial sums)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
    const float inv_l[2] = {l_run[0] > 0.f ? 1.0f / l_run[0] : 0.f, l_run[1] > 0.f ? 1.0f / l_run[1] : 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int qi = r0 + 8 * r;
        if (qi < a.Tq) {
            bf16* orow = a.out + (static_cast<size_t>(b) * a.Tq + qi) * a.ldo + h * D;
#pragma unroll
            for (int i = 2 * r; i < OR; i += 4)
                *reinterpret_cast<uint32_t*>(orow + frag_col(tw, i)) = pack_bf16x2(o[i] * inv_l[r], o[i + 1] * inv_l[r]);
        }
    }
}

template <int D, int NWG>
static int launch_attention(cudaStream_t stream, const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv,
                            const AttnArgs& a, int B) {
    using Cfg = AttnCfg<D, NWG>;
    auto kern = attention_kernel<D, NWG>;
    static DeviceOnce once;
    if (once.first()) {
        AF3_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    }
    dim3 grid(ceil_div(a.Tq, Cfg::BM), a.H, B);
    kern<<<grid, 128 * NWG, Cfg::SMEM_BYTES, stream>>>(mq, mk, mv, a);
    AF3_CHECK_LAUNCH();
    return 0;
}

int attention(cudaStream_t stream, const bf16* q, int ldq, const bf16* k, const bf16* v, int ldk, int kv_layout,
              int Tk_pitch, bf16* out, int ldo, int B, int H, int Hkv, int D, int Tq, int Tk, float scale, int causal,
              const int* kv_len, const int* kv_start) {
    AF3_REQUIRE(D == 64 || D == 128, "attention: head_dim must be 64 or 128");
    AF3_REQUIRE(H % Hkv == 0, "attention: H must be a multiple of Hkv");
    AF3_REQUIRE(ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0, "attention: output must be 16-byte aligned");
    if (B <= 0 || Tq <= 0) return 0;
    // one consumer warpgroup per CTA when AF3_ATTN_V1=1 asks for it (cross-check of the default two; read per call)
    const char* e1 = getenv("AF3_ATTN_V1");
    const int nwg = (e1 && e1[0] == '1') ? 1 : 2;
    const int bm = 64 * nwg;
    AttnArgs a{};
    a.Tq = Tq;
    a.Tk = Tk;
    a.H = H;
    a.Hkv = Hkv;
    a.causal = causal;
    a.kv_layout = kv_layout;
    a.scale_log2 = scale * LOG2E;
    a.kv_len = kv_len;
    a.kv_start = kv_start;
    a.out = out;
    a.ldo = ldo;
    CUtensorMap mq, mk, mv;
    if (int e = make_tmap_3d(&mq, q, (uint64_t)H * D, Tq, B, ldq, (uint64_t)Tq * ldq, 64, bm, 1)) return e;
    if (kv_layout) {
        if (int e = make_tmap_3d(&mk, k, D, Tk, (uint64_t)B * Hkv, ldk, (uint64_t)Tk_pitch * ldk, 64, AT_BN, 1)) return e;
        if (int e = make_tmap_3d(&mv, v, D, Tk, (uint64_t)B * Hkv, ldk, (uint64_t)Tk_pitch * ldk, 64, AT_BN, 1)) return e;
    } else {
        if (int e = make_tmap_3d(&mk, k, (uint64_t)Hkv * D, Tk, B, ldk, (uint64_t)Tk * ldk, 64, AT_BN, 1)) return e;
        if (int e = make_tmap_3d(&mv, v, (uint64_t)Hkv * D, Tk, B, ldk, (uint64_t)Tk * ldk, 64, AT_BN, 1)) return e;
    }
    if (D == 64) return nwg == 1 ? launch_attention<64, 1>(stream, mq, mk, mv, a, B) : launch_attention<64, 2>(stream, mq, mk, mv, a, B);
    return nwg == 1 ? launch_attention<128, 1>(stream, mq, mk, mv, a, B) : launch_attention<128, 2>(stream, mq, mk, mv, a, B);
}

}  // namespace af3
