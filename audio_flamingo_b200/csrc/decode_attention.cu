// Single-query (decode step) GQA attention over the pre-allocated KV cache; replaces SDPA at q_len = 1
// ([O] Q2M:227-238 -> SDPA:40-104) and the torch.cat cache growth (CACHE:119-120: the cache here is written in
// place by the qkv-projection epilogue / rope_kv_append).  HBM-bound: every K and V byte of the live context is read
// exactly once per step.
//
// One CTA = one (sequence, KV head, split) and serves all G = H/Hkv (<= 16) query heads sharing the KV head.  It streams
// its share of the live 128-key chunks through a 2-stage TMA ring (K and V tiles of 32 KB each, up to 128 KB in flight
// per SM) and keeps an online softmax, flash-decoding style.  The problem is transposed so that the 128 keys / 128
// output dims are the wgmma M dimension (two m64 halves) and the (padded) 16 query heads are N:
//     S^T[key, head] = K_tile[key, :] . Q[head, :]          wgmma m64n16k16 x 2 x 8,  A = K tile (K-major, via TMA)
//     O^T[dim, head] = V_tile^T[dim, key] . P^T[key, head]   wgmma m64n16k16 x 2 x 8,  A = V tile read MN-major
// so K and V never pass through registers.  Roles: warps 0-7 softmax + accumulation (thread = key row for S, = output dim row
// for O; the heads are split between two warp groups, see the kernel), warps 8-11 (one warpgroup) issue the MMAs and store
// the fp32 results to shared memory, warp 12 issues the TMA loads.  S, P and the per-chunk O are double-buffered so that
// S_{i+1} = K_{i+1} Q^T and the loads run ahead of softmax_i, and O_i is folded into the register accumulator after
// softmax_{i+1} has been handed to the tensor core.
// Splits: the host picks nz = min(chunks(Tmax), SMs / (B*Hkv)) so that B*Hkv*nz CTAs (one per SM, ~177 KB of smem) cover
// the GPU; the live chunk range [start/128, ceil(ctx/128)) of each sequence is divided evenly over the nz splits at run
// time.  nz == 1 (config 2: 32 x 4 = 128 CTAs) writes the normalised output directly; otherwise every split writes an
// (unnormalised o, max, sum) partial and the last-arriving split CTA of a (sequence, KV head) merges them (log-sum-exp
// combine) -- no separate combine kernel.
// ctx_len lives in device memory so the launch parameters are step-invariant (CUDA-graph replay).  Cache rows beyond
// the live context must hold finite values (the cache is zero-initialised): they are multiplied by P = 0.
// Algorithmic bytes per step: 2 (K,V) * Hkv * D * 2 B * ctx * B  (= 57344 B per token per sequence at 28 layers).
#include <stdlib.h>

#include "common.h"
#include "ptx.cuh"

namespace af3 {

constexpr int DA_CHUNK = 128;    // keys per ring stage
constexpr int DA_NH = 16;        // query heads per KV head, padded (UMMA N)
constexpr int DA_NS_MAX = 3;     // K/V ring stages (template parameter NS: 2 or 3)
constexpr int DA_THREADS = 416;  // warps 0-7: softmax / accumulate (thread = row x head group), warps 8-11: wgmma, warp 12: TMA
constexpr int DA_D = 128;
constexpr int DA_STAGE = 2 * DA_CHUNK * DA_D * 2;  // K tile + V tile
constexpr int DA_LD = DA_NH + 1;                   // row pitch (floats) of the S / O result tiles: conflict-free column reads
constexpr int da_smem(int ns) {
    return ns * DA_STAGE + 2 * (DA_NH * 128) /*Q: 2 blocks of 16 x 128 B*/ + 2 * 2 * (DA_NH * 128) /*P, double-buffered*/ +
           4 * 128 * DA_LD * 4 /*S, O: double-buffered [128][DA_LD] fp32*/ + 1024 /*align*/ + 2048 /*barriers + reduction scratch*/;
}

// N consecutive fp32 columns of one row of an S / O result tile
template <int N>
__device__ __forceinline__ void res_ldn(const float* p, uint32_t (&v)[N]) {
#pragma unroll
    for (int g = 0; g < N; ++g) v[g] = __float_as_uint(p[g]);
}

// Merge of the split partials of one (sequence, KV head), executed by the last-arriving split CTA.  Partial layout
// [b][h][split][D + 4] = (unnormalised o[D] relative to the split max, split max (log2 domain), split sum, pad).
// Work item = (head, 4 output dims): G * 32 items over the CTA's threads; the loads of all splits of an item are
// independent (two dependent rounds in total: maxima, then sums + outputs).  Only splits [s_lo, s_hi) hold live keys;
// the others never wrote theirs and are skipped by index.  Resets the arrival counter.
__device__ __forceinline__ void combine_heads(const float* __restrict__ part, bf16* __restrict__ out, int* counters, int b, int hk,
                                              int G, int H, int Hkv, int nsplit, int s_lo, int s_hi) {
    constexpr int D = DA_D, ST = D + 4, SB = 8;  // splits handled per unrolled block
    __threadfence();
    for (int item = threadIdx.x; item < G * (D / 4); item += blockDim.x) {
        const int g = item / (D / 4), dq = item % (D / 4);
        const int h = hk * G + g;
        const float* src = part + (static_cast<size_t>(b) * H + h) * nsplit * ST;
        float m = -INFINITY;
        for (int s0 = s_lo; s0 < s_hi; s0 += SB) {
            float ms[SB];
#pragma unroll
            for (int j = 0; j < SB; ++j) ms[j] = (s0 + j < s_hi) ? __ldcg(src + (s0 + j) * ST + D) : -INFINITY;
#pragma unroll
            for (int j = 0; j < SB; ++j) m = fmaxf(m, ms[j]);
        }
        float l = 0.f;
        float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s0 = s_lo; s0 < s_hi; s0 += SB) {
            float2 ml[SB];
            float4 ov[SB];
#pragma unroll
            for (int j = 0; j < SB; ++j) {
                const bool ok = s0 + j < s_hi;
                ml[j] = ok ? __ldcg(reinterpret_cast<const float2*>(src + (s0 + j) * ST + D)) : make_float2(-INFINITY, 0.f);
                ov[j] = ok ? __ldcg(reinterpret_cast<const float4*>(src + (s0 + j) * ST + dq * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int j = 0; j < SB; ++j) {
                const float w = (ml[j].x == -INFINITY) ? 0.f : exp2f(ml[j].x - m);
                l += w * ml[j].y;
                o.x += w * ov[j].x;
                o.y += w * ov[j].y;
                o.z += w * ov[j].z;
                o.w += w * ov[j].w;
            }
        }
        const float inv = l > 0.f ? 1.f / l : 0.f;
        bf16* dst = out + (static_cast<size_t>(b) * H + h) * D + dq * 4;
        *reinterpret_cast<uint2*>(dst) = make_uint2(pack_bf16x2(o.x * inv, o.y * inv), pack_bf16x2(o.z * inv, o.w * inv));
    }
    if (threadIdx.x == 0) counters[b * Hkv + hk] = 0;
}

// 2^x on the SFU (ex2.approx.ftz: relative error ~2^-22, far below the bf16 rounding of P); 2^-inf = +0
__device__ __forceinline__ float da_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// NG = padded query heads per KV head (8 when G <= 8, else 16).  The per-head loops are branch-free so the independent shuffle /
// SFU chains interleave.
// Two warp groups split the heads: warps 0-3 take heads [0, NG/2), warps 4-7 heads [NG/2, NG) of the same keys / output dims
// (warp w and w + 4 read the same rows of S / O): half the instructions per thread and chunk, two warps per scheduler, and the two
// groups only meet at the P hand-off (each has its own named barrier).
template <int NG, int DA_NS>
__global__ void __launch_bounds__(DA_THREADS, 1)
decode_attn_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                   const __grid_constant__ CUtensorMap map_v, float* __restrict__ part, bf16* __restrict__ out,
                   int* __restrict__ counters, int H, int Hkv, int nz, const int* __restrict__ ctx_len_p,
                   const int* __restrict__ kv_start, float scale_log2, unsigned long long* trace) {
    constexpr int D = DA_D;
    const int G = H / Hkv;
    const int b = blockIdx.x, hk = blockIdx.y, sp = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NH = NG / 2;  // heads per softmax thread
    if (tid == 0) trace_mark(trace, 0);
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sKV = smem;                         // DA_NS stages of {K: 2 blocks [128 keys x 128 B], V: same}
    uint8_t* sQ = sKV + DA_NS * DA_STAGE;        // 2 blocks [16 heads x 128 B]
    uint8_t* sP = sQ + 2 * DA_NH * 128;          // 2 buffers x 2 blocks [16 heads x 128 B]  (64 keys along each 128-byte row)
    uint64_t* bars = reinterpret_cast<uint64_t*>(sP + 4 * DA_NH * 128);
    uint64_t *q_full = bars, *k_full = bars + 1, *v_full = k_full + DA_NS_MAX, *kv_empty = v_full + DA_NS_MAX,
             *s_full = kv_empty + DA_NS_MAX, *p_full = s_full + 2, *o_full = p_full + 2;
    float* red = reinterpret_cast<float*>(bars) + 256;  // [2 parities][4 warps][16 heads] chunk maxima, then [4][16] sums
    float* sS = reinterpret_cast<float*>(bars) + 512;   // S^T results [2][128 keys][DA_LD], then O^T results [2][128 dims][DA_LD]
    float* sO = sS + 2 * 128 * DA_LD;
    __shared__ int last_flag;

    // ---- prologue (no global-memory reads: overlaps the tail of the previous kernel under PDL)
    if (tid == 384) {
        tma_prefetch_desc(&map_q);
        tma_prefetch_desc(&map_k);
        tma_prefetch_desc(&map_v);
        mbar_init(q_full, 1);
        for (int s = 0; s < DA_NS; ++s) {
            mbar_init(k_full + s, 1);
            mbar_init(v_full + s, 1);
            mbar_init(kv_empty + s, 4);   // one arrival per wgmma warp
        }
        for (int s = 0; s < 2; ++s) {
            mbar_init(s_full + s, 128);
            mbar_init(p_full + s, 256);
            mbar_init(o_full + s, 128);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    if (warp == 12 && lane == 0) {
        // Before the dependency resolves: ask L2 for this CTA's K/V chunks.  Only a hint -- nothing is read into the SM, so it does not
        // matter that ctx_len may still hold the previous step's value or that the row the q/k/v projection is appending right now is
        // not there yet (its write lands in the same L2 line; the real loads below come after griddepcontrol.wait).
        const int ctx0 = *reinterpret_cast<const volatile int*>(ctx_len_p);
        const int start0 = kv_start ? kv_start[b] : 0;
        const int lo0 = start0 / DA_CHUNK, hi0 = (ctx0 + DA_CHUNK - 1) / DA_CHUNK;
        const int live0 = max(hi0 - lo0, 0), cps0 = (live0 + nz - 1) / nz;
        const int beg0 = lo0 + sp * cps0, n0 = max(min(hi0, beg0 + cps0) - beg0, 0);
        for (int i = 0; i < n0; ++i) {
            const int row = (beg0 + i) * DA_CHUNK;
#pragma unroll
            for (int db = 0; db < 2; ++db) {
                tma_prefetch_l2_3d(&map_k, db * 64, row, b * Hkv + hk);
                tma_prefetch_l2_3d(&map_v, db * 64, row, b * Hkv + hk);
            }
        }
    }
    pdl_wait();
    if (tid == 0) trace_mark(trace, 1);

    // ---- this CTA's share of the live chunks
    const int ctx = *ctx_len_p;
    const int start = kv_start ? kv_start[b] : 0;
    const int c_lo = start / DA_CHUNK, c_hi = (ctx + DA_CHUNK - 1) / DA_CHUNK;
    const int n_live = max(c_hi - c_lo, 0);
    const int cps = (n_live + nz - 1) / nz;                    // chunks per split
    const int n_used = cps > 0 ? (n_live + cps - 1) / cps : 0;  // splits that hold live keys
    const int c_beg = c_lo + sp * cps;
    const int n = max(min(c_hi, c_beg + cps) - c_beg, 0);

    if (n > 0) {
        if (warp == 12) {
            if (lane == 0) {
                mbar_arrive_expect_tx(q_full, 2 * DA_NH * 128);
#pragma unroll
                for (int db = 0; db < 2; ++db) tma_load_2d(sQ + db * DA_NH * 128, &map_q, q_full, db * 64, b * (H + 2 * Hkv) + hk * G);
                for (int i = 0; i < n; ++i) {
                    const int s = i % DA_NS;
                    if (i >= DA_NS) mbar_wait(kv_empty + s, ((i / DA_NS) - 1) & 1);
                    uint8_t* st = sKV + s * DA_STAGE;
                    const int row = (c_beg + i) * DA_CHUNK;
                    mbar_arrive_expect_tx(k_full + s, DA_CHUNK * D * 2);
#pragma unroll
                    for (int db = 0; db < 2; ++db) tma_load_3d(st + db * 16384, &map_k, k_full + s, db * 64, row, b * Hkv + hk);
                    mbar_arrive_expect_tx(v_full + s, DA_CHUNK * D * 2);
#pragma unroll
                    for (int db = 0; db < 2; ++db) tma_load_3d(st + 32768 + db * 16384, &map_v, v_full + s, db * 64, row, b * Hkv + hk);
                }
            }
            __syncwarp();
        } else if (warp >= 8) {
            // ---- wgmma warpgroup: each product is two m64 halves (keys / output dims [0, 64) and [64, 128)); the fp32 results
            //      go to the S / O tiles in shared memory, rows = keys / output dims, columns = heads
            const int tw = tid - 256;
            const uint32_t aKV = smem_u32(sKV), aQ = smem_u32(sQ), aP = smem_u32(sP);
            auto store = [&](float* dst, float (&r)[2][8]) {
#pragma unroll
                for (int mh = 0; mh < 2; ++mh)
#pragma unroll
                    for (int e = 0; e < 8; ++e) dst[(mh * 64 + frag_row(tw, e)) * DA_LD + frag_col(tw, e)] = r[mh][e];
            };
            // O^T_j = V_j^T . P_j^T  (fresh accumulator: the running output lives in the softmax warps' registers)
            auto issue_pv = [&](int j) {
                const int s = j % DA_NS;
                mbar_wait(p_full + (j & 1), (j >> 1) & 1);
                mbar_wait(v_full + s, (j / DA_NS) & 1);
                const uint32_t aV = aKV + s * DA_STAGE + 32768, aPj = aP + (j & 1) * (2 * DA_NH * 128);
                float r[2][8];
                wgmma_fence();
#pragma unroll
                for (int mh = 0; mh < 2; ++mh)
#pragma unroll
                    for (int kk = 0; kk < DA_CHUNK / 16; ++kk)
                        wgmma_m64n16_ss<1, 0>(r[mh], make_smem_desc_sw128(aV + mh * 16384 + kk * 2048, 16384, 1024),
                                              make_smem_desc_sw128(aPj + (kk >> 2) * (DA_NH * 128) + (kk & 3) * 32, 0, 1024), kk != 0);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(r[0]);
                fence_regs(r[1]);
                if (lane == 0) mbar_arrive(kv_empty + s);
                store(sO + (j & 1) * 128 * DA_LD, r);
                mbar_arrive(o_full + (j & 1));
            };
            mbar_wait(q_full, 0);
            for (int i = 0; i < n; ++i) {
                const int s = i % DA_NS;
                // S^T_i = K_i . Q^T into S[i & 1]: that buffer was last read by softmax_{i-2}, whose P the previous
                // iteration's issue_pv(i - 2) has already waited for
                mbar_wait(k_full + s, (i / DA_NS) & 1);
                const uint32_t aK = aKV + s * DA_STAGE;
                float r[2][8];
                wgmma_fence();
#pragma unroll
                for (int mh = 0; mh < 2; ++mh)
#pragma unroll
                    for (int kk = 0; kk < D / 16; ++kk)
                        wgmma_m64n16_ss<0, 0>(r[mh], make_smem_desc_sw128(aK + mh * 64 * 128 + (kk >> 2) * 16384 + (kk & 3) * 32, 0, 1024),
                                              make_smem_desc_sw128(aQ + (kk >> 2) * (DA_NH * 128) + (kk & 3) * 32, 0, 1024), kk != 0);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(r[0]);
                fence_regs(r[1]);
                store(sS + (i & 1) * 128 * DA_LD, r);
                mbar_arrive(s_full + (i & 1));
                if (i >= 1) issue_pv(i - 1);
            }
            issue_pv(n - 1);
        } else {
            // ---- online softmax: thread = key (row of S) for S, = output dim for O; columns = heads [hg * NH, hg * NH + NH)
            const int wq = warp & 3, hg = warp >> 2;
            const int kt = wq * 32 + lane;  // key within the chunk / output dim
            const int col_off = hg * NH;
            const int bar_id = 1 + hg;      // named barrier of this head group's four warps
            float m_run[NH], m_prev[NH], m_pp[NH], l_thr[NH], acc[NH];
#pragma unroll
            for (int g = 0; g < NH; ++g) {
                m_run[g] = -INFINITY;   // running max after the current chunk
                m_prev[g] = -INFINITY;  // ... one chunk back (what O_{i-1} is relative to)
                m_pp[g] = -INFINITY;    // ... two chunks back (what acc is relative to when O_{i-1} is folded in)
                l_thr[g] = 0.f;         // this key lane's share of the softmax denominator
                acc[g] = 0.f;           // this output dim's running numerator
            }
            if (hg == 0) {   // P rows of heads >= NG are never written again: zero them once in both buffers
                const int kc = kt & 63;
#pragma unroll
                for (int pb = 0; pb < 2; ++pb) {
                    uint8_t* blk = sP + pb * (2 * DA_NH * 128) + (kt >> 6) * (DA_NH * 128);
#pragma unroll
                    for (int g = NG; g < DA_NH; ++g)
                        *reinterpret_cast<bf16*>(blk + g * 128 + ((((kc >> 3) ^ (g & 7)) << 4) | ((kc & 7) << 1))) = __float2bfloat16_rn(0.f);
                }
            }
            // acc is relative to m_from (the running max at its last update); O_j is relative to m_to
            auto accumulate = [&](int j, const float (&m_from)[NH], const float (&m_to)[NH]) {
                mbar_wait(o_full + (j & 1), (j >> 1) & 1);
                uint32_t ov[NH];
                res_ldn<NH>(sO + ((j & 1) * 128 + kt) * DA_LD + col_off, ov);
#pragma unroll
                for (int g = 0; g < NH; ++g) {
                    const float a = (m_from[g] == -INFINITY) ? 0.f : da_exp2(m_from[g] - m_to[g]);
                    acc[g] = fmaf(acc[g], a, __uint_as_float(ov[g]));
                }
            };
            for (int i = 0; i < n; ++i) {
                const int j = (c_beg + i) * DA_CHUNK + kt;
                const bool valid = j >= start && j < ctx;
                float* redm = red + (i & 1) * 64;
                mbar_wait(s_full + (i & 1), (i >> 1) & 1);
                uint32_t sv[NH];
                res_ldn<NH>(sS + ((i & 1) * 128 + kt) * DA_LD + col_off, sv);
                float t[NH], mx[NH];
#pragma unroll
                for (int g = 0; g < NH; ++g) {
                    t[g] = (valid && hg * NH + g < G) ? __uint_as_float(sv[g]) * scale_log2 : -INFINITY;
                    mx[g] = t[g];
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
                    for (int g = 0; g < NH; ++g) mx[g] = fmaxf(mx[g], __shfl_xor_sync(0xffffffffu, mx[g], o));
                }
                if (lane < NH) {  // lane g publishes head g's warp maximum (all lanes hold it after the butterfly)
                    float v = mx[0];
#pragma unroll
                    for (int g = 1; g < NH; ++g) v = (lane == g) ? mx[g] : v;
                    redm[wq * DA_NH + col_off + lane] = v;
                }
                asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
                uint8_t* blk = sP + (i & 1) * (2 * DA_NH * 128) + (kt >> 6) * (DA_NH * 128);
                const int kc = kt & 63;
#pragma unroll
                for (int g = 0; g < NH; ++g) {
                    const int gh = col_off + g;  // head within the KV group
                    const float mc = fmaxf(fmaxf(redm[gh], redm[DA_NH + gh]), fmaxf(redm[2 * DA_NH + gh], redm[3 * DA_NH + gh]));
                    const float m_new = fmaxf(m_run[g], mc);
                    const float a = (m_run[g] == -INFINITY) ? 0.f : da_exp2(m_run[g] - m_new);
                    const float p = (t[g] == -INFINITY) ? 0.f : da_exp2(t[g] - m_new);  // masked keys / padded heads -> 0
                    l_thr[g] = fmaf(l_thr[g], a, p);
                    m_pp[g] = m_prev[g];
                    m_prev[g] = m_run[g];
                    m_run[g] = m_new;
                    // P^T[key = kt][head gh] -> B tile [16 heads][128 keys], K-major, 128B swizzle: row gh, key column kt
                    *reinterpret_cast<bf16*>(blk + gh * 128 + ((((kc >> 3) ^ (gh & 7)) << 4) | ((kc & 7) << 1))) = __float2bfloat16_rn(p);
                }
                fence_proxy_async_smem();
                mbar_arrive(p_full + (i & 1));
                // fold in the previous chunk's P.V (relative to m_prev = running max after chunk i-1)
                if (i >= 1) accumulate(i - 1, m_pp, m_prev);
            }
            accumulate(n - 1, m_prev, m_run);
            if (tid == 0) trace_mark(trace, 2);
            // ---- softmax denominators: sum the per-thread partial sums over the 128 key lanes
            float* reds = red + 128;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
                for (int g = 0; g < NH; ++g) l_thr[g] += __shfl_xor_sync(0xffffffffu, l_thr[g], o);
            }
            if (lane < NH) {
                float v = l_thr[0];
#pragma unroll
                for (int g = 1; g < NH; ++g) v = (lane == g) ? l_thr[g] : v;
                reds[wq * DA_NH + col_off + lane] = v;
            }
            asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
#pragma unroll
            for (int g = 0; g < NH; ++g) {
                const int gh = col_off + g;
                if (gh < G) {
                    const float L = reds[gh] + reds[DA_NH + gh] + reds[2 * DA_NH + gh] + reds[3 * DA_NH + gh];
                    if (nz == 1) {
                        out[(static_cast<size_t>(b) * H + hk * G + gh) * D + kt] = __float2bfloat16_rn(L > 0.f ? acc[g] / L : 0.f);
                    } else {
                        float* dst = part + ((static_cast<size_t>(b) * H + hk * G + gh) * nz + sp) * (D + 4);
                        dst[kt] = acc[g];
                        if (kt == 0) {
                            dst[D] = m_run[g];
                            dst[D + 1] = L;
                        }
                    }
                }
            }
        }
    }
    if (nz > 1) __threadfence();  // partials visible before this split is counted
    __syncthreads();
    if (nz == 1) {
        if (tid == 0) trace_mark(trace, 3);
        return;
    }
    // ---- the last-arriving split CTA of this (sequence, KV head) merges all split partials (log-sum-exp combine):
    //      replaces a separate combine kernel per layer
    if (tid == 0) last_flag = (atomicAdd(counters + b * Hkv + hk, 1) == nz - 1);
    __syncthreads();
    if (last_flag) combine_heads(part, out, counters, b, hk, G, H, Hkv, nz, 0, n_used);
    if (tid == 0) trace_mark(trace, 3);
}

static int n_chunks(int Tmax) { return ceil_div(Tmax, DA_CHUNK); }

// splits per (sequence, KV head): enough CTAs to cover the SMs, never more than there are chunks.  AF3_DECODE_SPLITS
// overrides (tests).
static int pick_splits(int B, int Hkv, int Tmax) {
    int nz = sm_count() / (B * Hkv);
    if (const char* e = getenv("AF3_DECODE_SPLITS")) {
        const int v = atoi(e);
        if (v > 0) nz = v;
    }
    return nz < 1 ? 1 : (nz > n_chunks(Tmax) ? n_chunks(Tmax) : nz);
}

// scratch = split partials (sized for the maximum split count) + one arrival counter per (sequence, KV head); the
// counters must be ZERO on first use (the kernel leaves them zero)
static size_t partial_bytes(int B, int H, int D, int Tmax) {
    return (static_cast<size_t>(B) * H * n_chunks(Tmax) * (D + 4) * sizeof(float) + 255) & ~static_cast<size_t>(255);
}
size_t decode_attention_scratch_bytes(int B, int H, int D, int Tmax) {
    return partial_bytes(B, H, D, Tmax) + static_cast<size_t>(B) * H * sizeof(int);
}

int decode_attention(cudaStream_t stream, const bf16* qkv, const bf16* k_cache, const bf16* v_cache, bf16* out,
                     float* scratch, int B, int H, int Hkv, int D, int Tmax, const int* ctx_len, const int* kv_start,
                     float scale) {
    AF3_REQUIRE(D == 128, "decode_attention: head_dim must be 128");
    AF3_REQUIRE(H % Hkv == 0 && H / Hkv <= DA_NH, "decode_attention: at most 16 query heads per KV head");
    AF3_REQUIRE(ctx_len != nullptr, "decode_attention: ctx_len must be a device pointer");
    AF3_REQUIRE(Hkv <= 65535, "decode_attention: too many KV heads");
    const int nz = pick_splits(B, Hkv, Tmax);
    // ring depth 2 (128 KB in flight): a third stage does not fit next to the S / O result tiles in 227 KB
    constexpr int ns = 2;
    static_assert(da_smem(ns) <= 232448, "shared memory per CTA");
    static DeviceOnce once;
    if (once.first()) {
        AF3_CHECK_CUDA(cudaFuncSetAttribute(decode_attn_kernel<8, ns>, cudaFuncAttributeMaxDynamicSharedMemorySize, da_smem(ns)));
        AF3_CHECK_CUDA(cudaFuncSetAttribute(decode_attn_kernel<16, ns>, cudaFuncAttributeMaxDynamicSharedMemorySize, da_smem(ns)));
    }
    CUtensorMap mq, mk, mv;
    // q heads as rows of 128: the packed projection row of sequence b holds (H + 2 Hkv) such rows
    if (int e = make_tmap_2d(&mq, qkv, D, static_cast<uint64_t>(B) * (H + 2 * Hkv), D, 64, DA_NH)) return e;
    if (int e = make_tmap_3d(&mk, k_cache, D, Tmax, static_cast<uint64_t>(B) * Hkv, D, static_cast<uint64_t>(Tmax) * D, 64,
                             DA_CHUNK, 1))
        return e;
    if (int e = make_tmap_3d(&mv, v_cache, D, Tmax, static_cast<uint64_t>(B) * Hkv, D, static_cast<uint64_t>(Tmax) * D, 64,
                             DA_CHUNK, 1))
        return e;
    dim3 grid(B, Hkv, nz);
    int* counters = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(scratch) + partial_bytes(B, H, D, Tmax));
    auto kern = (H / Hkv <= 8) ? decode_attn_kernel<8, ns> : decode_attn_kernel<16, ns>;
    AF3_CHECK_CUDA(launch_kernel(kern, grid, dim3(DA_THREADS), da_smem(ns), stream, mq, mk, mv, scratch, out, counters, H, Hkv, nz,
                                 ctx_len, kv_start, scale * 1.4426950408889634f, trace_next_slot()));
    return 0;
}

}  // namespace af3
