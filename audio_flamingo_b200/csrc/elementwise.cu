// HBM-bound CUDA-core kernels of the AF3 path: LayerNorm, AvgPool+LayerNorm, RMSNorm, conv-stem im2col,
// rotary embedding + KV-cache append, embedding gather / audio-row scatter, gate/up weight packing, argmax, FP8 activation
// quantization.
// All bf16 tensors are accessed with 16-byte vector loads/stores, one warp (or a few) per row, fp32 statistics,
// and the reference's bf16 rounding points are reproduced op by op (cited per kernel).
#include "common.h"
#include "ptx.cuh"

#include <cuda_fp8.h>

namespace af3 {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 t = __bfloat1622float2(h[e]);
        f[2 * e] = t.x;
        f[2 * e + 1] = t.y;
    }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

constexpr int NORM_MAXV = 16;  // uint4 chunks per lane -> dim <= 4096

// ---------------------------------------------------------------------------------------------------------
// FP8 activation quantization (include/af3b200.h af3_quant_fp8), the input side of the FP8 decoder projections that
// replaces the activation quantization of [O] integrations/finegrained_fp8.py FP8Linear.forward.  Per row and 128-column
// group: amax = max |x| (fp32, exact from bf16), s = amax / 448 rounded to nearest (s = 1 for an all-zero group),
// q = e4m3(x / s) rounded to nearest even with saturation -- torch's (x.float() / s).to(torch.float8_e4m3fn) bit for bit.
// One warp per row and pair of groups: each half-warp owns one group, 16-byte loads (8 bf16) and 8-byte stores per lane.
// q: [rows][K] e4m3 (pitch K); scales: [K / 128][rows] fp32, so that a GEMM's k-block reads the scales of consecutive
// tokens from consecutive addresses.
__global__ void __launch_bounds__(256)
quant_fp8_kernel(const bf16* __restrict__ x, int ldx, uint8_t* __restrict__ q, float* __restrict__ scales, int rows, int K,
                 unsigned long long* trace) {
    if (threadIdx.x == 0) trace_mark(trace, 0);
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) trace_mark(trace, 1);
    const int pairs = (K + 255) >> 8;
    const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (w < rows * pairs) {  // warp-uniform: every lane takes part in the shuffles
        const int row = w / pairs;
        const int col = ((w - row * pairs) << 8) + lane * 8;
        const bool ok = col < K;
        float f[8];
        unpack8(ok ? __ldcs(reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * ldx + col)) : make_uint4(0, 0, 0, 0), f);
        float amax = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) amax = fmaxf(amax, fabsf(f[e]));
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));  // within the half-warp
        const float s = amax > 0.f ? __fdiv_rn(amax, 448.f) : 1.f;
        uint32_t packed[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(f[4 * h], s), __fdiv_rn(f[4 * h + 1], s)),
                                                                     __NV_SATFINITE, __NV_E4M3);
            const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(f[4 * h + 2], s), __fdiv_rn(f[4 * h + 3], s)),
                                                                     __NV_SATFINITE, __NV_E4M3);
            packed[h] = static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
        }
        if (ok) {
            *reinterpret_cast<uint2*>(q + static_cast<size_t>(row) * K + col) = make_uint2(packed[0], packed[1]);
            if ((lane & 15) == 0) scales[static_cast<size_t>(col >> 7) * rows + row] = s;
        }
    }
    if (threadIdx.x == 0) trace_mark(trace, 3);
}

int quant_fp8(cudaStream_t stream, const bf16* x, int ldx, uint8_t* q, float* scales, int rows, int K) {
    AF3_REQUIRE(rows > 0 && K > 0 && K % 128 == 0, "quant_fp8: K must be a positive multiple of 128");
    AF3_REQUIRE(ldx >= K && ldx % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(q) & 7) == 0,
                "quant_fp8: x must be 16-byte aligned with a pitch that is a multiple of 8 elements, q 8-byte aligned");
    const long long warps = static_cast<long long>(rows) * ((K + 255) / 256);
    AF3_CHECK_CUDA(launch_kernel(quant_fp8_kernel, dim3(static_cast<unsigned>((warps + 7) / 8)), dim3(256), 0, stream, x, ldx, q, scales,
                                 rows, K, trace_next_slot()));
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// LayerNorm ([O] AF3M:224,232,366: nn.LayerNorm, eps 1e-5; fp32 statistics, one rounding to bf16).
// POOL: the row is first formed as bf16((x[2t] + x[2t+1]) / 2)  (nn.AvgPool1d(2,2), AF3M:364-365).
template <bool POOL, int NV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, const bf16* __restrict__ gamma,
                 const bf16* __restrict__ beta, int rows, int dim, float eps, int T_in, int T_out) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int nchunk = dim >> 3;
    float v[NV][8];
    float sum = 0.f;
    size_t in_row = row;
    if (POOL) {
        const int w = row / T_out, t = row - w * T_out;
        in_row = static_cast<size_t>(w) * T_in + 2 * t;
    }
    const uint4* xp = reinterpret_cast<const uint4*>(x + in_row * dim);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = lane + 32 * i;
        if (c < nchunk) {
            unpack8(__ldcs(xp + c), v[i]);   // streaming: the row is read once per launch
            if (POOL) {
                float b[8];
                unpack8(__ldcs(xp + c + nchunk), b);
#pragma unroll
                for (int e = 0; e < 8; ++e) v[i][e] = bf16_round((v[i][e] + b[e]) * 0.5f);
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) sum += v[i][e];
        }
    }
    const float mean = warp_sum(sum) / dim;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = lane + 32 * i;
        if (c < nchunk) {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float d = v[i][e] - mean;
                sq += d * d;
            }
        }
    }
    const float rstd = rsqrtf(warp_sum(sq) / dim + eps);
    uint4* yp = reinterpret_cast<uint4*>(y + static_cast<size_t>(row) * dim);
    const uint4* gp = reinterpret_cast<const uint4*>(gamma);
    const uint4* bp = reinterpret_cast<const uint4*>(beta);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = lane + 32 * i;
        if (c < nchunk) {
            float g[8], b[8], o[8];
            unpack8(__ldg(gp + c), g);
            unpack8(__ldg(bp + c), b);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] = (v[i][e] - mean) * rstd * g[e] + b[e];
            yp[c] = pack8(o);   // default policy: the next GEMM reads y right away (L2)
        }
    }
}

// NV = 16-byte chunks per lane: sized to the row so the row lives in few registers (occupancy = bandwidth here)
template <bool POOL>
static int launch_layernorm(cudaStream_t stream, const bf16* x, bf16* y, const bf16* gamma, const bf16* beta, int rows, int dim,
                            float eps, int T_in, int T_out) {
    const int need = ceil_div(dim >> 3, 32);
    dim3 grid(ceil_div(rows, 8)), block(256);
#define AF3_LN_CASE(NV)                                                                                              \
    if (need <= NV) {                                                                                                \
        layernorm_kernel<POOL, NV><<<grid, block, 0, stream>>>(x, y, gamma, beta, rows, dim, eps, T_in, T_out);      \
        AF3_CHECK_LAUNCH();                                                                                          \
        return 0;                                                                                                    \
    }
    AF3_LN_CASE(2)
    AF3_LN_CASE(5)
    AF3_LN_CASE(8)
    AF3_LN_CASE(16)
#undef AF3_LN_CASE
    return fail("layernorm: dim too large");
}

int layernorm(cudaStream_t stream, const bf16* x, bf16* y, const bf16* gamma, const bf16* beta, int rows, int dim,
              float eps) {
    AF3_REQUIRE(dim % 8 == 0 && dim <= NORM_MAXV * 256, "layernorm: dim must be a multiple of 8 and <= 4096");
    if (rows <= 0) return 0;
    return launch_layernorm<false>(stream, x, y, gamma, beta, rows, dim, eps, 0, 0);
}
int avgpool_layernorm(cudaStream_t stream, const bf16* x, bf16* y, const bf16* gamma, const bf16* beta, int n_win,
                      int T, int dim, float eps) {
    AF3_REQUIRE(dim % 8 == 0 && dim <= NORM_MAXV * 256, "avgpool_layernorm: dim must be a multiple of 8 and <= 4096");
    const int T_out = T / 2;
    const int rows = n_win * T_out;
    if (rows <= 0) return 0;
    return launch_layernorm<true>(stream, x, y, gamma, beta, rows, dim, eps, T, T_out);
}

// ---------------------------------------------------------------------------------------------------------
// Qwen2RMSNorm ([O] Q2M:258-263): h = x.float(); h = h * rsqrt(mean(h^2) + eps); return weight * h.to(bf16).
// Many rows (prefill): one warp per row.  The row is held PACKED (bf16, 4 registers per 16-byte chunk) and unpacked twice --
// once for the sum of squares, once for the output -- instead of once into 8 fp32 registers per chunk: for the 3584-wide
// decoder that is 56 instead of 112 live registers per thread, which doubles the resident warps per SM.  Round 1 measured this
// kernel at 0.37 of the HBM peak (ncu: 127 registers, 16 warps per SM): every warp loads its whole row, reduces, then stores,
// so the bytes in flight per SM are (resident warps) x (row bytes) x (share of a warp's life spent loading) -- occupancy IS the
// bandwidth here.  x is read with the streaming hint (read once per launch).
template <int NV>
__global__ void __launch_bounds__(256)
rmsnorm_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, const bf16* __restrict__ weight, int rows, int dim,
               float eps, const int* __restrict__ row_idx, unsigned long long* trace) {
    if (threadIdx.x == 0) trace_mark(trace, 0);
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) trace_mark(trace, 1);
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const size_t in_row = row_idx ? static_cast<size_t>(row_idx[row]) : static_cast<size_t>(row);
    const int nchunk = dim >> 3;
    const uint4* xp = reinterpret_cast<const uint4*>(x + in_row * dim);
    uint4 xr[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = lane + 32 * i;
        xr[i] = (c < nchunk) ? __ldcs(xp + c) : make_uint4(0, 0, 0, 0);
    }
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        float f[8];
        unpack8(xr[i], f);
#pragma unroll
        for (int e = 0; e < 8; ++e) sq += f[e] * f[e];
    }
    const float rstd = rsqrtf(warp_sum(sq) / dim + eps);
    // opaque to the optimiser: without this the first unpack is kept alive (8 fp32 registers per chunk) instead of redone
#pragma unroll
    for (int i = 0; i < NV; ++i) asm volatile("" : "+r"(xr[i].x), "+r"(xr[i].y), "+r"(xr[i].z), "+r"(xr[i].w));
    uint4* yp = reinterpret_cast<uint4*>(y + static_cast<size_t>(row) * dim);
    const uint4* wp = reinterpret_cast<const uint4*>(weight);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = lane + 32 * i;
        if (c < nchunk) {
            float f[8], w[8], o[8];
            unpack8(xr[i], f);
            unpack8(__ldg(wp + c), w);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] = w[e] * bf16_round(f[e] * rstd);
            yp[c] = pack8(o);   // default policy: the GEMM that follows re-reads y, part of it still in L2
        }
    }
    if (threadIdx.x == 0) trace_mark(trace, 3);
}

// Few rows (decode step: 32 tokens): one CTA of 256 threads per row, so a 7 KB row is a single round of 16-byte loads
// per thread instead of 14 dependent-latency rounds in one warp.
__global__ void __launch_bounds__(256)
rmsnorm_rowblock_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, const bf16* __restrict__ weight, int dim, float eps,
                        const int* __restrict__ row_idx, unsigned long long* trace) {
    if (threadIdx.x == 0) trace_mark(trace, 0);
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) trace_mark(trace, 1);
    const int row = blockIdx.x;
    const size_t in_row = row_idx ? static_cast<size_t>(row_idx[row]) : static_cast<size_t>(row);
    const int nchunk = dim >> 3;
    const uint4* xp = reinterpret_cast<const uint4*>(x + in_row * dim);
    const uint4* wp = reinterpret_cast<const uint4*>(weight);
    constexpr int MAXC = 4;  // dim <= 8192
    float v[MAXC][8], w[MAXC][8];
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < MAXC; ++i) {
        const int c = threadIdx.x + 256 * i;
        if (c < nchunk) {
            unpack8(xp[c], v[i]);
            unpack8(__ldg(wp + c), w[i]);
#pragma unroll
            for (int e = 0; e < 8; ++e) sq += v[i][e] * v[i][e];
        }
    }
    __shared__ float part[8];
    sq = warp_sum(sq);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = sq;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) tot += part[i];
    const float rstd = rsqrtf(tot / dim + eps);
    uint4* yp = reinterpret_cast<uint4*>(y + static_cast<size_t>(row) * dim);
#pragma unroll
    for (int i = 0; i < MAXC; ++i) {
        const int c = threadIdx.x + 256 * i;
        if (c < nchunk) {
            float o[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] = w[i][e] * bf16_round(v[i][e] * rstd);
            yp[c] = pack8(o);
        }
    }
    if (threadIdx.x == 0) trace_mark(trace, 3);
}

int rmsnorm(cudaStream_t stream, const bf16* x, bf16* y, const bf16* weight, int rows, int dim, float eps,
            const int* row_idx) {
    AF3_REQUIRE(dim % 8 == 0 && dim <= NORM_MAXV * 256, "rmsnorm: dim must be a multiple of 8 and <= 4096");
    if (rows <= 0) return 0;
    if (rows <= 1024) {
        AF3_CHECK_CUDA(launch_kernel(rmsnorm_rowblock_kernel, dim3(rows), dim3(256), 0, stream, x, y, weight, dim, eps, row_idx, trace_next_slot()));
        return 0;
    }
    const int need = ceil_div(dim >> 3, 32);
    unsigned long long* tr = trace_next_slot();
    if (need <= 5)
        AF3_CHECK_CUDA(launch_kernel(rmsnorm_kernel<5>, dim3(ceil_div(rows, 8)), dim3(256), 0, stream, x, y, weight, rows, dim, eps, row_idx, tr));
    else if (need <= 14)
        AF3_CHECK_CUDA(launch_kernel(rmsnorm_kernel<14>, dim3(ceil_div(rows, 8)), dim3(256), 0, stream, x, y, weight, rows, dim, eps, row_idx, tr));
    else
        AF3_CHECK_CUDA(launch_kernel(rmsnorm_kernel<16>, dim3(ceil_div(rows, 8)), dim3(256), 0, stream, x, y, weight, rows, dim, eps, row_idx, tr));
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// conv1 im2col ([O] AF3M:343: conv1d(k=3, pad=1) over [n_win, C, T]): cols[(w,t)][kk*C + c] = bf16(x[w][c][t+kk-1]).
// A CTA transposes a [C x 64(+2)] slab through shared memory: reads coalesced along t, writes 16 B along c.
template <typename TIn>
__global__ void __launch_bounds__(256)
im2col_conv1_kernel(const TIn* __restrict__ in, bf16* __restrict__ cols, int C, int T) {
    extern __shared__ bf16 tile[];  // [C][66 + 2 pad]
    constexpr int TB = 64, P = 68;
    const int w = blockIdx.y, t0 = blockIdx.x * TB;
    const TIn* xin = in + static_cast<size_t>(w) * C * T;
    for (int i = threadIdx.x; i < C * (TB + 2); i += blockDim.x) {
        const int c = i / (TB + 2), tt = i - c * (TB + 2);
        const int t = t0 + tt - 1;
        float v = 0.f;
        if (t >= 0 && t < T) v = static_cast<float>(xin[static_cast<size_t>(c) * T + t]);
        tile[c * P + tt] = __float2bfloat16_rn(v);
    }
    __syncthreads();
    const int cpr = 3 * C / 8;  // uint4 chunks per output row
    for (int i = threadIdx.x; i < TB * cpr; i += blockDim.x) {
        const int tl = i / cpr, ch = i - tl * cpr;
        const int t = t0 + tl;
        if (t >= T) continue;
        const int kk = (ch * 8) / C, c0 = ch * 8 - kk * C;
        uint32_t pk[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const bf16 a = tile[(c0 + 2 * e) * P + tl + kk];
            const bf16 b = tile[(c0 + 2 * e + 1) * P + tl + kk];
            pk[e] = static_cast<uint32_t>(__bfloat16_as_ushort(a)) | (static_cast<uint32_t>(__bfloat16_as_ushort(b)) << 16);
        }
        reinterpret_cast<uint4*>(cols + (static_cast<size_t>(w) * T + t) * 3 * C)[ch] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
    }
}

int im2col_conv1(cudaStream_t stream, const void* in, int in_is_f32, bf16* cols, int n_win, int C, int T) {
    AF3_REQUIRE(C % 8 == 0, "im2col_conv1: C must be a multiple of 8");
    if (n_win <= 0) return 0;
    dim3 grid(ceil_div(T, 64), n_win);
    const size_t smem = static_cast<size_t>(C) * 68 * sizeof(bf16);
    if (in_is_f32)
        im2col_conv1_kernel<float><<<grid, 256, smem, stream>>>(static_cast<const float*>(in), cols, C, T);
    else
        im2col_conv1_kernel<bf16><<<grid, 256, smem, stream>>>(static_cast<const bf16*>(in), cols, C, T);
    AF3_CHECK_LAUNCH();
    return 0;
}

// conv2 im2col ([O] AF3M:344: conv1d(k=3, stride=2, pad=1)) on the channel-last activation [n_win*T, C]:
// output row (w, t') is the concatenation of input rows 2t'-1, 2t', 2t'+1 (zero outside [0, T)).
__global__ void __launch_bounds__(256)
im2col_conv2_kernel(const bf16* __restrict__ in, bf16* __restrict__ cols, int C, int T, int T_out, long long total16) {
    const int cpr = 3 * C / 8;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total16;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long row = i / cpr;
        const int ch = static_cast<int>(i - row * cpr);
        const int w = static_cast<int>(row / T_out), tp = static_cast<int>(row - static_cast<long long>(w) * T_out);
        const int kk = (ch * 8) / C, c0 = ch * 8 - kk * C;
        const int t = 2 * tp + kk - 1;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (t >= 0 && t < T) v = *reinterpret_cast<const uint4*>(in + (static_cast<size_t>(w) * T + t) * C + c0);
        reinterpret_cast<uint4*>(cols)[i] = v;
    }
}

int im2col_conv2(cudaStream_t stream, const bf16* in, bf16* cols, int n_win, int C, int T) {
    AF3_REQUIRE(C % 8 == 0, "im2col_conv2: C must be a multiple of 8");
    const int T_out = (T - 1) / 2 + 1;
    const long long total16 = static_cast<long long>(n_win) * T_out * (3 * C / 8);
    if (total16 <= 0) return 0;
    const int grid = static_cast<int>(((total16 + 255) / 256) < 132ll * 16 ? ((total16 + 255) / 256) : 132ll * 16);
    im2col_conv2_kernel<<<grid, 256, 0, stream>>>(in, cols, C, T, T_out, total16);
    AF3_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// gate/up interleave for the fused SwiGLU GEMM: per 128 features, 128 gate rows then 128 up rows (zero padded).
__global__ void pack_gate_up_kernel(const bf16* __restrict__ gate, const bf16* __restrict__ up, bf16* __restrict__ packed,
                                    int F, int K, long long total16) {
    const int cpr = K / 8;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total16;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long prow = i / cpr;
        const int ch = static_cast<int>(i - prow * cpr);
        const int blk = static_cast<int>(prow / 256), within = static_cast<int>(prow % 256);
        const int f = blk * 128 + (within & 127);
        uint4 v = make_uint4(0, 0, 0, 0);
        if (f < F) v = reinterpret_cast<const uint4*>((within < 128 ? gate : up) + static_cast<size_t>(f) * K)[ch];
        reinterpret_cast<uint4*>(packed)[i] = v;
    }
}
int pack_gate_up(cudaStream_t stream, const bf16* gate, const bf16* up, bf16* packed, int F, int K) {
    AF3_REQUIRE(K % 8 == 0, "pack_gate_up: K must be a multiple of 8");
    const long long total16 = 2ll * ceil_div(F, 128) * 128 * (K / 8);
    const int grid = static_cast<int>(((total16 + 255) / 256) < 132ll * 16 ? ((total16 + 255) / 256) : 132ll * 16);
    pack_gate_up_kernel<<<grid, 256, 0, stream>>>(gate, up, packed, F, K, total16);
    AF3_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// Rotary embedding + KV append ([O] Q2M:100-146 rotate-half RoPE with fp32 tables cast to bf16; CACHE:119-120).
// Every bf16 op of the reference rounds: q*cos, rotate_half(q)*sin and their sum are each rounded to bf16.
// HEAD_PAR = false (prefill): one thread = one (token, 8-wide d chunk of the first half); cos/sin are computed once and
// reused for every head.  HEAD_PAR = true (decode, few tokens): one thread = one (token, head, chunk) so the few
// tokens still spread over thousands of threads instead of a 32-iteration dependent loop per thread.
// All accesses are 16-byte vectors (chunk d..d+7 and its rotate-half partner d+D/2..d+D/2+7).
template <bool HEAD_PAR>
__global__ void __launch_bounds__(256)
rope_kv_append_kernel(bf16* __restrict__ qkv, bf16* __restrict__ k_cache, bf16* __restrict__ v_cache, int B, int T,
                      int H, int Hkv, int D, int Tmax, int pos0, const int* __restrict__ pos0_dev,
                      const int* __restrict__ kv_start, const float* __restrict__ inv_freq) {
    const int half = D >> 1;
    const int cpt = half >> 3;  // 8-wide chunks per token half
    const int heads = H + 2 * Hkv;
    const long long total = static_cast<long long>(B) * T * cpt * (HEAD_PAR ? heads : 1);
    pdl_launch_dependents();
    pdl_wait();
    const int p0 = pos0_dev ? *pos0_dev : pos0;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        long long rest = i;
        int h_only = 0;
        if (HEAD_PAR) {
            h_only = static_cast<int>(rest % heads);
            rest /= heads;
        }
        const int ch = static_cast<int>(rest % cpt);
        const long long bt = rest / cpt;
        const int t = static_cast<int>(bt % T);
        const int b = static_cast<int>(bt / T);
        const int d0 = ch * 8;
        const int cpos = p0 + t;  // cache slot
        if (cpos >= Tmax) continue;  // never past the allocation (device-side position: the host cannot check it)
        bf16* tok = qkv + static_cast<size_t>(bt) * heads * D;
        const int h_beg = HEAD_PAR ? h_only : 0, h_end = HEAD_PAR ? h_only + 1 : heads;
        if (h_beg < H + Hkv) {
            int pos = cpos - (kv_start ? kv_start[b] : 0);
            if (pos < 0) pos = 1;  // padded slot: position_ids.masked_fill_(mask == 0, 1) (GEN:721)
            float c[8], sn[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float fr = inv_freq[d0 + e] * static_cast<float>(pos);
                c[e] = bf16_round(cosf(fr));
                sn[e] = bf16_round(sinf(fr));
            }
            for (int h = h_beg; h < min(h_end, H + Hkv); ++h) {
                bf16* row = tok + static_cast<size_t>(h) * D;
                float x1[8], x2[8], o1[8], o2[8];
                unpack8(*reinterpret_cast<const uint4*>(row + d0), x1);
                unpack8(*reinterpret_cast<const uint4*>(row + d0 + half), x2);
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    o1[e] = bf16_round(bf16_round(x1[e] * c[e]) + bf16_round(-x2[e] * sn[e]));
                    o2[e] = bf16_round(bf16_round(x2[e] * c[e]) + bf16_round(x1[e] * sn[e]));
                }
                bf16* dst = row;
                if (h >= H) dst = k_cache + ((static_cast<size_t>(b) * Hkv + (h - H)) * Tmax + cpos) * D;
                *reinterpret_cast<uint4*>(dst + d0) = pack8(o1);
                *reinterpret_cast<uint4*>(dst + d0 + half) = pack8(o2);
            }
        }
        for (int h = max(h_beg, H + Hkv); h < h_end; ++h) {  // value heads: plain copy into the cache
            const int hk = h - H - Hkv;
            const bf16* row = tok + static_cast<size_t>(h) * D;
            bf16* dst = v_cache + ((static_cast<size_t>(b) * Hkv + hk) * Tmax + cpos) * D;
            *reinterpret_cast<uint4*>(dst + d0) = *reinterpret_cast<const uint4*>(row + d0);
            *reinterpret_cast<uint4*>(dst + d0 + half) = *reinterpret_cast<const uint4*>(row + d0 + half);
        }
    }
}

int rope_kv_append(cudaStream_t stream, bf16* qkv, bf16* k_cache, bf16* v_cache, int B, int T, int H, int Hkv, int D,
                   int Tmax, int pos0, const int* pos0_dev, const int* kv_start, const float* inv_freq) {
    AF3_REQUIRE(D % 16 == 0 && inv_freq, "rope: head dim must be a multiple of 16 / missing inv_freq");
    AF3_REQUIRE(pos0_dev || pos0 + T <= Tmax, "rope: KV cache overflow");
    const long long tok_chunks = static_cast<long long>(B) * T * (D / 16);
    if (tok_chunks <= 0) return 0;
    const bool head_par = tok_chunks < 8192;  // decode steps / short prompts
    const long long total = tok_chunks * (head_par ? (H + 2 * Hkv) : 1);
    const int grid = static_cast<int>(((total + 255) / 256) < 132ll * 32 ? ((total + 255) / 256) : 132ll * 32);
    if (head_par)
        AF3_CHECK_CUDA(launch_kernel(rope_kv_append_kernel<true>, dim3(grid), dim3(256), 0, stream, qkv, k_cache, v_cache, B, T, H,
                                     Hkv, D, Tmax, pos0, pos0_dev, kv_start, inv_freq));
    else
        AF3_CHECK_CUDA(launch_kernel(rope_kv_append_kernel<false>, dim3(grid), dim3(256), 0, stream, qkv, k_cache, v_cache, B, T, H,
                                     Hkv, D, Tmax, pos0, pos0_dev, kv_start, inv_freq));
    return 0;
}

// Music Flamingo rotary TIME embedding on the AF-Whisper output ([O] transformers/models/musicflamingo/
// modular_musicflamingo.py:167-227: rotate_half on interleaved pairs, MusicFlamingoRotaryEmbedding.forward, and
// apply_rotary_time_emb which computes in fp64).  x bf16 [W*T, dim] in place; the first 4*n_freq features are rotated:
//   features [0, 2 n_freq)        : window axis, freq = (round(ts[w,0] / window_duration) / max_len) * inv_freq[j/2]
//   features [2 n_freq, 4 n_freq) : time axis,   freq = ((t / max_len) * 2 pi) * inv_freq[(j - 2 n_freq)/2]
// each multiplied by angle = -ts[w,t] * 2 * pi, all in fp32 exactly in the reference's operation order; cos/sin in fp32,
// the rotation itself in fp64, one rounding back to bf16.  One thread per (row, pair).
__global__ void __launch_bounds__(256)
rotary_time_kernel(bf16* __restrict__ x, const float* __restrict__ ts, const float* __restrict__ inv_freq, int W, int T, int dim,
                   int n_freq, float window_duration, float max_len) {
    const long long total = static_cast<long long>(W) * T * 2 * n_freq;
    const float two_pi = static_cast<float>(2.0 * 3.141592653589793);
    const float pi_f = static_cast<float>(3.141592653589793);
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int p = static_cast<int>(i % (2 * n_freq));  // pair index: features 2p, 2p+1
        const long long row = i / (2 * n_freq);
        const int t = static_cast<int>(row % T), w = static_cast<int>(row / T);
        float freq;
        if (p < n_freq) {
            const float wpos = rintf(ts[static_cast<size_t>(w) * T] / window_duration) / max_len;
            freq = wpos * inv_freq[p];
        } else {
            const float pos = (static_cast<float>(t) / max_len) * two_pi;
            freq = pos * inv_freq[p - n_freq];
        }
        const float angle = ((-ts[row]) * 2.0f) * pi_f;
        const float f = freq * angle;
        const double c = static_cast<double>(cosf(f)), s = static_cast<double>(sinf(f));
        bf16* px = x + row * dim + 2 * p;
        const double x0 = static_cast<double>(__bfloat162float(px[0])), x1 = static_cast<double>(__bfloat162float(px[1]));
        px[0] = __double2bfloat16(x0 * c + (-x1) * s);
        px[1] = __double2bfloat16(x1 * c + x0 * s);
    }
}

int rotary_time(cudaStream_t stream, bf16* x, const float* ts, const float* inv_freq, int W, int T, int dim, int n_freq,
                float window_duration, float max_len) {
    AF3_REQUIRE(4 * n_freq <= dim && n_freq > 0, "rotary_time: rotary width exceeds the feature dim");
    const long long total = static_cast<long long>(W) * T * 2 * n_freq;
    if (total <= 0) return 0;
    const int grid = static_cast<int>(((total + 255) / 256) < 132ll * 16 ? ((total + 255) / 256) : 132ll * 16);
    rotary_time_kernel<<<grid, 256, 0, stream>>>(x, ts, inv_freq, W, T, dim, n_freq, window_duration, max_len);
    AF3_CHECK_LAUNCH();
    return 0;
}

// Flamingo-style gated residual ([O] transformers/models/idefics/modeling_idefics.py:796-806, the executable analogue of AF2's
// gated xattn-dense block, SURVEY 8-f.4):  out = resid + tanh(alpha) * y   with every bf16 op of the reference rounded:
// t = bf16(tanh(alpha)), p = bf16(t * y), out = bf16(resid + p).  alpha: bf16 [dim] (alpha_type "vector") or one value
// (alpha_scalar != 0, alpha_type "float").  row_gate (optional, int32 [rows]): rows whose gate is 0 take y = 0 (tokens that attend
// to no media, idefics:797).  One warp per row, 16-byte accesses.
__global__ void __launch_bounds__(256)
gated_residual_kernel(const bf16* __restrict__ resid, const bf16* __restrict__ y, const bf16* __restrict__ alpha, int alpha_scalar,
                      const int* __restrict__ row_gate, bf16* __restrict__ out, int rows, int dim) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const bool open = row_gate ? (row_gate[row] != 0) : true;
    const uint4* rp = reinterpret_cast<const uint4*>(resid + static_cast<size_t>(row) * dim);
    const uint4* yp = reinterpret_cast<const uint4*>(y + static_cast<size_t>(row) * dim);
    uint4* op = reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * dim);
    const float t_scalar = alpha_scalar ? bf16_round(tanhf(__bfloat162float(alpha[0]))) : 0.f;
    for (int c = lane; c < dim / 8; c += 32) {
        float r[8], v[8], a8[8], o[8];
        unpack8(rp[c], r);
        unpack8(yp[c], v);
        if (!alpha_scalar) unpack8(__ldg(reinterpret_cast<const uint4*>(alpha) + c), a8);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float t = alpha_scalar ? t_scalar : bf16_round(tanhf(a8[e]));
            const float p = bf16_round(t * (open ? v[e] : 0.f));
            o[e] = r[e] + p;
        }
        op[c] = pack8(o);
    }
}

int gated_residual(cudaStream_t stream, const bf16* resid, const bf16* y, const bf16* alpha, int alpha_scalar, const int* row_gate,
                   bf16* out, int rows, int dim) {
    AF3_REQUIRE(dim % 8 == 0 && alpha, "gated_residual: dim must be a multiple of 8 and alpha given");
    if (rows <= 0) return 0;
    gated_residual_kernel<<<ceil_div(rows, 8), 256, 0, stream>>>(resid, y, alpha, alpha_scalar, row_gate, out, rows, dim);
    AF3_CHECK_LAUNCH();
    return 0;
}

// cos/sin table of ONE decode step for the RoPE-fused q/k/v projection epilogue: cs[b][i] = (bf16(cos), bf16(sin)) of
// inv_freq[i] * position(b), position = slot - kv_start[b] (Q2M:100-113; identical for all layers of the step).
__global__ void rope_table_kernel(float2* __restrict__ cs, int B, int half, const int* __restrict__ pos_dev,
                                  const int* __restrict__ kv_start, const float* __restrict__ inv_freq, unsigned long long* trace) {
    if (threadIdx.x == 0) trace_mark(trace, 0);
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) trace_mark(trace, 1);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * half) return;
    const int b = i / half, d = i - b * half;
    int pos = *pos_dev - (kv_start ? kv_start[b] : 0);
    if (pos < 0) pos = 1;
    const float fr = inv_freq[d] * static_cast<float>(pos);
    cs[i] = make_float2(bf16_round(cosf(fr)), bf16_round(sinf(fr)));
    if (threadIdx.x == 0) trace_mark(trace, 3);
}

int rope_table(cudaStream_t stream, float* cs, int B, int D, const int* pos_dev, const int* kv_start, const float* inv_freq) {
    AF3_REQUIRE(D % 2 == 0 && pos_dev && inv_freq, "rope_table: bad arguments");
    const int n = B * (D / 2);
    if (n <= 0) return 0;
    AF3_CHECK_CUDA(launch_kernel(rope_table_kernel, dim3(ceil_div(n, 256)), dim3(256), 0, stream, reinterpret_cast<float2*>(cs), B,
                                 D / 2, pos_dev, kv_start, inv_freq, trace_next_slot()));
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// Embedding gather + audio scatter ([O] AF3M:557 embed_tokens; :469-473 valid-frame select; :563-566 masked_scatter).
// Kernel 1 (one CTA): exclusive scan of (ids == audio_token_id) over the flattened prompt -> ordinal of each audio
// token; exclusive scan of post_len -> first ordinal of each window.  Kernel 2: one warp per token row copy.
__global__ void __launch_bounds__(1024)
scatter_index_kernel(const int64_t* __restrict__ ids, int n_tok, int64_t audio_id, const int* __restrict__ post_len,
                     int n_win, int frames, int* __restrict__ src_row /*[n_tok]*/, int* __restrict__ counts,
                     unsigned long long* trace) {
    __shared__ int warp_tot[32];
    __shared__ int carry;
    __shared__ int win_base[1025];
    if (threadIdx.x == 0) trace_mark(trace, 0);
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) trace_mark(trace, 1);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // window prefix (n_win <= 1024 handled in one sweep; larger handled serially by thread 0)
    if (tid == 0) {
        int acc = 0;
        for (int w = 0; w < n_win; ++w) {
            if (w < 1025) win_base[w] = acc;
            acc += min(post_len[w], frames);
        }
        counts[1] = acc;
        carry = 0;
    }
    __syncthreads();
    for (int base = 0; base < n_tok; base += 1024) {
        const int i = base + tid;
        const int flag = (i < n_tok && ids[i] == audio_id) ? 1 : 0;
        int incl = flag;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int n = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += n;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int v = warp_tot[lane], inc2 = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int n = __shfl_up_sync(0xffffffffu, inc2, o);
                if (lane >= o) inc2 += n;
            }
            warp_tot[lane] = inc2 - v;  // exclusive
            if (lane == 31) win_base[1024] = inc2;  // block total (scratch slot)
        }
        __syncthreads();
        const int ord = carry + warp_tot[warp] + incl - flag;
        if (i < n_tok) {
            int row = -1;
            if (flag) {
                // binary search the window whose [base, base+len) contains ord
                int lo = 0, hi = n_win - 1;
                while (lo < hi) {
                    const int mid = (lo + hi + 1) >> 1;
                    if (win_base[mid] <= ord) lo = mid; else hi = mid - 1;
                }
                const int off = ord - win_base[lo];
                row = (off < min(post_len[lo], frames)) ? lo * frames + off : -2;  // -2: more tokens than features
            }
            src_row[i] = row;
        }
        __syncthreads();
        if (tid == 0) carry += win_base[1024];
        __syncthreads();
    }
    if (tid == 0) counts[0] = carry;
    if (tid == 0) trace_mark(trace, 3);
}

__global__ void __launch_bounds__(256)
embed_scatter_kernel(const int64_t* __restrict__ ids, int n_tok, const bf16* __restrict__ table, int dim,
                     const bf16* __restrict__ audio, const int* __restrict__ src_row, bf16* __restrict__ out,
                     unsigned long long* trace) {
    if (threadIdx.x == 0) trace_mark(trace, 0);
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) trace_mark(trace, 1);
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n_tok) return;
    const int sr = src_row[row];
    const bf16* src = (sr >= 0) ? audio + static_cast<size_t>(sr) * dim : table + static_cast<size_t>(ids[row]) * dim;
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    uint4* d4 = reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * dim);
    for (int c = lane; c < dim / 8; c += 32) d4[c] = __ldg(s4 + c);
    if (threadIdx.x == 0) trace_mark(trace, 3);
}

int embed_scatter(cudaStream_t stream, const int64_t* ids, int n_tok, const bf16* table, int dim, int64_t audio_id,
                  const bf16* audio, int n_win, int frames, const int* post_len, bf16* out, int* src_row_scratch,
                  int* counts) {
    AF3_REQUIRE(dim % 8 == 0, "embed_scatter: dim must be a multiple of 8");
    AF3_REQUIRE(n_win <= 1024, "embed_scatter: at most 1024 windows per call");
    if (n_tok <= 0) return 0;
    static const int zero_len = 0;
    (void)zero_len;
    AF3_CHECK_CUDA(launch_kernel(scatter_index_kernel, dim3(1), dim3(1024), 0, stream, ids, n_tok, audio_id, post_len, n_win,
                                 frames, src_row_scratch, counts, trace_next_slot()));
    AF3_CHECK_CUDA(launch_kernel(embed_scatter_kernel, dim3(ceil_div(n_tok, 8)), dim3(256), 0, stream, ids, n_tok, table, dim,
                                 audio, src_row_scratch, out, trace_next_slot()));
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// Greedy argmax over fp32 logits ([O] GEN:2762 logits.float(), :2793 torch.argmax -> first maximal index).
// Two stages so that the 19.5 MB of logits at batch 32 are read by B x 32 CTAs (not B): stage 1 reduces a slice of the
// row to (max, first index), stage 2 merges the 32 slices.  NaNs are ignored; an all-NaN row yields 0.
constexpr int AM_SPLIT = 32;

__device__ __forceinline__ void argmax_merge(float& best, int& bi, float ob, int oi) {
    if (ob > best || (ob == best && oi < bi)) {
        best = ob;
        bi = oi;
    }
}

__global__ void __launch_bounds__(256)
argmax_partial_kernel(const float* __restrict__ logits, int V, float* __restrict__ pmax, int* __restrict__ pidx,
                      unsigned long long* trace) {
    if (threadIdx.x == 0) trace_mark(trace, 0);
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) trace_mark(trace, 1);
    const int row = blockIdx.x, sp = blockIdx.y;
    const float* p = logits + static_cast<size_t>(row) * V;
    const int per = ((V + AM_SPLIT - 1) / AM_SPLIT + 3) & ~3;  // slice length, multiple of 4
    const int beg = sp * per, end = min(V, beg + per);
    float best = -INFINITY;
    int bi = 0x7fffffff;
    const bool vec = (reinterpret_cast<uintptr_t>(p) & 15) == 0;
    if (vec) {
        const int n4 = max(end - beg, 0) / 4;
        const float4* p4 = reinterpret_cast<const float4*>(p + beg);
        for (int i = threadIdx.x; i < n4; i += blockDim.x) {
            const float4 v = __ldg(p4 + i);
            const int base = beg + 4 * i;
            argmax_merge(best, bi, v.x, base);
            argmax_merge(best, bi, v.y, base + 1);
            argmax_merge(best, bi, v.z, base + 2);
            argmax_merge(best, bi, v.w, base + 3);
        }
        for (int i = beg + n4 * 4 + threadIdx.x; i < end; i += blockDim.x) argmax_merge(best, bi, p[i], i);
    } else {
        for (int i = beg + threadIdx.x; i < end; i += blockDim.x) argmax_merge(best, bi, p[i], i);
    }
    __shared__ float sb[8];
    __shared__ int si[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) argmax_merge(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
    if ((threadIdx.x & 31) == 0) {
        sb[threadIdx.x >> 5] = best;
        si[threadIdx.x >> 5] = bi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) argmax_merge(best, bi, sb[w], si[w]);
        pmax[row * AM_SPLIT + sp] = best;
        pidx[row * AM_SPLIT + sp] = bi;
        trace_mark(trace, 3);
    }
}

__global__ void __launch_bounds__(32)
argmax_final_kernel(const float* __restrict__ pmax, const int* __restrict__ pidx, int64_t* __restrict__ out,
                    unsigned long long* trace) {
    if (threadIdx.x == 0) trace_mark(trace, 0);
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) trace_mark(trace, 1);
    const int row = blockIdx.x, lane = threadIdx.x;
    float best = pmax[row * AM_SPLIT + lane];
    int bi = pidx[row * AM_SPLIT + lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) argmax_merge(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
    if (lane == 0) out[row] = (bi == 0x7fffffff) ? 0 : bi;
    if (lane == 0) trace_mark(trace, 3);
}

size_t argmax_scratch_bytes(int B) { return static_cast<size_t>(B) * AM_SPLIT * (sizeof(float) + sizeof(int)); }

int argmax(cudaStream_t stream, const float* logits, int B, int V, int64_t* out, void* scratch) {
    if (B <= 0) return 0;
    AF3_REQUIRE(scratch != nullptr, "argmax: scratch of af3_argmax_scratch_bytes(B) bytes required");
    float* pmax = static_cast<float*>(scratch);
    int* pidx = reinterpret_cast<int*>(pmax + static_cast<size_t>(B) * AM_SPLIT);
    AF3_CHECK_CUDA(launch_kernel(argmax_partial_kernel, dim3(B, AM_SPLIT), dim3(256), 0, stream, logits, V, pmax, pidx, trace_next_slot()));
    AF3_CHECK_CUDA(launch_kernel(argmax_final_kernel, dim3(B), dim3(32), 0, stream, static_cast<const float*>(pmax),
                                 static_cast<const int*>(pidx), out, trace_next_slot()));
    return 0;
}

// One token of the greedy loop's bookkeeping, on the device ([O] GEN:2797-2805): pad rows that have finished, append the token,
// hand it to the next step's embedding lookup, update the unfinished mask with the EOS set and publish "every row finished".
// Inside the captured decode step this replaces five small torch launches per token between graph replays.
//   ctl[0] = number of EOS ids (0: no EOS handling), ctl[1] = pad id;  gen_idx = index of the token being appended (advanced here).
__global__ void __launch_bounds__(256)
token_step_kernel(const int64_t* __restrict__ raw_ids, int B, int* __restrict__ unfinished, const int64_t* __restrict__ eos,
                  const int64_t* __restrict__ ctl, int64_t* __restrict__ tok_buf, int cap, int* __restrict__ gen_idx,
                  int64_t* __restrict__ ids_out, int* __restrict__ done_flags, unsigned long long* trace) {
    if (threadIdx.x == 0) trace_mark(trace, 0);
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) trace_mark(trace, 1);
    __shared__ int any_unfinished;
    if (threadIdx.x == 0) any_unfinished = 0;
    __syncthreads();
    const int i = *gen_idx;
    const int n_eos = static_cast<int>(ctl[0]);
    const int64_t pad = ctl[1];
    int mine = 0;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        int64_t t = raw_ids[b];
        int u = 1;
        if (n_eos > 0) {
            u = unfinished[b];
            if (!u) t = pad;                                   // GEN:2797
            for (int e = 0; e < n_eos; ++e) u = (t == eos[e]) ? 0 : u;   // GEN:2803 (EosTokenCriteria)
            unfinished[b] = u;
        }
        if (i < cap) tok_buf[static_cast<size_t>(b) * cap + i] = t;
        ids_out[b] = t;
        mine |= u;
    }
    if (mine) any_unfinished = 1;   // benign race: every writer stores 1
    __syncthreads();
    if (threadIdx.x == 0) {
        if (i < cap) done_flags[i] = (n_eos > 0 && !any_unfinished) ? 1 : 0;   // GEN:2805
        *gen_idx = i + 1;
        trace_mark(trace, 3);
    }
}

int token_step(cudaStream_t stream, const int64_t* raw_ids, int B, int* unfinished, const int64_t* eos, const int64_t* ctl,
               int64_t* tok_buf, int cap, int* gen_idx, int64_t* ids_out, int* done_flags) {
    if (B <= 0) return 0;
    AF3_REQUIRE(raw_ids && unfinished && eos && ctl && tok_buf && gen_idx && ids_out && done_flags && cap > 0, "token_step: null argument");
    AF3_CHECK_CUDA(launch_kernel(token_step_kernel, dim3(1), dim3(256), 0, stream, raw_ids, B, unfinished, eos, ctl, tok_buf, cap, gen_idx, ids_out,
                                 done_flags, trace_next_slot()));
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// Greedy logits processors + selection (include/af3b200.h af3_logits_process_argmax), the device restatement of
// [O] generation/logits_process.py SequenceBias, NoRepeatNGram, NoBadWords, MinLength, MinNewTokensLength, ForcedEOSToken,
// SuppressTokens and SuppressTokensAtBegin in the order of [O] generation/utils.py _get_logits_processor.
// Per row and step the processed value of token t is
//   forced step  : 0 at the forced EOS ids (unless suppressed or begin-suppressed), -inf elsewhere
//   otherwise    : -inf if any mask rule hits t, else x + bias_total(t)
// Rules that depend on only the token (single-token bias, single-token bad words, suppress_tokens) sit in a dense fp32
// vector static_add [V] (bias, or -inf); the rest depend on the history or the step and are found by logits_rules_kernel,
// which writes a short per-row list of (token, kind, value).  logits_process_partial_kernel then reads each logit once,
// adds static_add, overrides the listed tokens and reduces its slice to (max, first index) exactly like
// argmax_partial_kernel; argmax_final_kernel merges the slices.  The list order is irrelevant to every output: mask bits are
// OR-ed, a token has at most one ADD / SET entry, and (max, first index) merging is order-free.
enum : int {
    LP_S = 0, LP_NGRAM, LP_MINLEN, LP_MINNEW, LP_BEGIN, LP_FORCED, LP_STATIC,
    LP_NEOS, LP_OEOS, LP_NBEGIN, LP_OBEGIN, LP_NFORCED, LP_OFORCED, LP_NBAD, LP_OBAD, LP_NGRP, LP_OGRP,
    LP_HDR = 32
};
enum : int { LP_MASK = 0, LP_ADD = 1, LP_SET = 2 };
constexpr int LP_MAXW = 1024;   // bitmap words per slice -> slices of up to 32768 tokens

__device__ __forceinline__ int64_t lp_hist(const int64_t* __restrict__ prompt, const int64_t* __restrict__ gen, size_t off, int S,
                                           int t) {
    return t < S ? __ldg(prompt + off + t) : gen[off + (t - S)];
}

__device__ __forceinline__ void lp_emit(int2* __restrict__ list, int cap, int* cnt, int tok, int kind, float val) {
    const int s = atomicAdd(cnt, 1);   // slot allocation only; see the order note above
    if (s < cap) list[s] = make_int2(static_cast<int>(static_cast<unsigned>(tok) | (static_cast<unsigned>(kind) << 30)), __float_as_int(val));
}

// One CTA per row.  History = prompt[b][0, S) followed by generated[b][0, *gen_idx): the input_ids the reference's processors see.
__global__ void __launch_bounds__(256)
logits_rules_kernel(const int64_t* __restrict__ prompt, const int64_t* __restrict__ generated, int ld, int V, const int* __restrict__ gen_idx,
                    const int* __restrict__ tab, int2* __restrict__ list, int2* __restrict__ row_info, int cap, unsigned long long* trace) {
    if (threadIdx.x == 0) trace_mark(trace, 0);
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) trace_mark(trace, 1);
    __shared__ int h[LP_HDR];
    __shared__ int cnt;
    if (threadIdx.x < LP_HDR) h[threadIdx.x] = tab[threadIdx.x];
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    const int b = blockIdx.x;
    const int S = h[LP_S], gen = *gen_idx, cur = S + gen;
    const size_t off = static_cast<size_t>(b) * ld;
    int2* out = list + static_cast<size_t>(b) * cap;
    const bool forced = h[LP_FORCED] >= 0 && cur == h[LP_FORCED];
    const bool begin = cur == h[LP_BEGIN];
    if (forced) {   // ForcedEOSToken assigns the row; only SuppressTokens / SuppressTokensAtBegin come after it
        for (int r = threadIdx.x; r < h[LP_NFORCED]; r += blockDim.x) {
            const int* f = tab + h[LP_OFORCED] + 2 * r;
            const bool sup = (f[1] & 1) || ((f[1] & 2) && begin);
            lp_emit(out, cap, &cnt, f[0], LP_SET, sup ? -INFINITY : 0.f);
        }
    } else {
        // NoRepeatNGram: every earlier n-gram whose first n-1 tokens equal the last n-1 tokens bans its last token
        const int n = h[LP_NGRAM];
        if (n > 0 && cur + 1 >= n) {
            const int p0 = cur - n + 1;
            for (int j = threadIdx.x; j <= cur - n; j += blockDim.x) {
                bool hit = true;
                for (int k = 0; k < n - 1 && hit; ++k) hit = lp_hist(prompt, generated, off, S, j + k) == lp_hist(prompt, generated, off, S, p0 + k);
                if (hit) {
                    const int64_t t = lp_hist(prompt, generated, off, S, j + n - 1);
                    if (t >= 0 && t < V) lp_emit(out, cap, &cnt, static_cast<int>(t), LP_MASK, -INFINITY);
                }
            }
        }
        // NoBadWords, sequences of 2+ tokens: the last token is banned when the history ends with the others
        for (int r = threadIdx.x; r < h[LP_NBAD]; r += blockDim.x) {
            const int* rec = tab + h[LP_OBAD] + 2 * r;
            const int* seq = tab + rec[0];
            const int L = rec[1];
            if (L > cur) continue;
            bool hit = true;
            for (int k = 0; k < L - 1 && hit; ++k) hit = lp_hist(prompt, generated, off, S, cur - L + 1 + k) == seq[k];
            if (hit) lp_emit(out, cap, &cnt, seq[L - 1], LP_MASK, -INFINITY);
        }
        // SequenceBias, sequences of 2+ tokens, grouped by last token: 0 + single-token bias + every matching sequence's bias
        // in dict order, one fp32 add each (the reference's bias tensor accumulation)
        for (int r = threadIdx.x; r < h[LP_NGRP]; r += blockDim.x) {
            const int* g = tab + h[LP_OGRP] + 4 * r;
            float total = 0.f + __int_as_float(g[1]);
            bool any = false;
            for (int m = 0; m < g[3]; ++m) {
                const int* mem = tab + g[2] + 3 * m;
                const int* seq = tab + mem[0];
                const int L = mem[1];
                if (L > cur) continue;
                bool hit = true;
                for (int k = 0; k < L - 1 && hit; ++k) hit = lp_hist(prompt, generated, off, S, cur - L + 1 + k) == seq[k];
                if (hit) {
                    total += __int_as_float(mem[2]);
                    any = true;
                }
            }
            if (any) lp_emit(out, cap, &cnt, g[0], LP_ADD, total);
        }
        // MinLength (counts the prompt) and MinNewTokensLength (counts generated tokens) mask the EOS ids
        if (cur < h[LP_MINLEN] || gen < h[LP_MINNEW])
            for (int r = threadIdx.x; r < h[LP_NEOS]; r += blockDim.x) lp_emit(out, cap, &cnt, tab[h[LP_OEOS] + r], LP_MASK, -INFINITY);
        if (begin)
            for (int r = threadIdx.x; r < h[LP_NBEGIN]; r += blockDim.x) lp_emit(out, cap, &cnt, tab[h[LP_OBEGIN] + r], LP_MASK, -INFINITY);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        row_info[b] = make_int2(min(cnt, cap), forced ? 1 : 0);
        trace_mark(trace, 3);
    }
}

__global__ void __launch_bounds__(256)
logits_process_partial_kernel(const float* __restrict__ logits, int V, const float* __restrict__ static_add, const int* __restrict__ tab,
                              const int2* __restrict__ list, const int2* __restrict__ row_info, int cap, float* __restrict__ scores,
                              float* __restrict__ pmax, int* __restrict__ pidx, unsigned long long* trace) {
    if (threadIdx.x == 0) trace_mark(trace, 0);
    pdl_launch_dependents();
    __shared__ unsigned ovr[LP_MAXW];   // token of the slice has a list entry
    __shared__ unsigned msk[LP_MAXW];   // ... and one of them is a mask
    const int row = blockIdx.x, sp = blockIdx.y;
    const int per = ((V + AM_SPLIT - 1) / AM_SPLIT + 3) & ~3;
    const int beg = sp * per, end = min(V, beg + per);
    const int nw = (per + 31) >> 5;
    for (int w = threadIdx.x; w < nw; w += blockDim.x) ovr[w] = msk[w] = 0u;
    pdl_wait();
    if (threadIdx.x == 0) trace_mark(trace, 1);
    const bool has_static = tab[LP_STATIC] != 0;
    const int2 info = row_info[row];
    const int n = info.x;
    const bool forced = info.y != 0;
    const int2* ent = list + static_cast<size_t>(row) * cap;
    __syncthreads();
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
        const int2 en = ent[e];
        const int t = en.x & 0x3fffffff;
        if (t < beg || t >= end) continue;
        const unsigned bit = 1u << ((t - beg) & 31);
        atomicOr(&ovr[(t - beg) >> 5], bit);
        if ((static_cast<unsigned>(en.x) >> 30) == LP_MASK) atomicOr(&msk[(t - beg) >> 5], bit);
    }
    __syncthreads();
    const float* p = logits + static_cast<size_t>(row) * V;
    float* so = scores ? scores + static_cast<size_t>(row) * V : nullptr;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    const bool vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(so) | reinterpret_cast<uintptr_t>(static_add)) & 15) == 0;
    int tail = beg;
    if (vec) {
        const int n4 = max(end - beg, 0) / 4;
        for (int i = threadIdx.x; i < n4; i += blockDim.x) {
            const int rel = 4 * i, base = beg + rel;
            const unsigned skip = (ovr[rel >> 5] >> (rel & 31)) & 0xFu;
            float4 v = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
            if (!forced) {
                v = __ldg(reinterpret_cast<const float4*>(p + base));
                if (has_static) {
                    const float4 s = __ldg(reinterpret_cast<const float4*>(static_add + base));
                    v = make_float4(v.x + s.x, v.y + s.y, v.z + s.z, v.w + s.w);
                }
            }
            if (!(skip & 1u)) argmax_merge(best, bi, v.x, base);
            if (!(skip & 2u)) argmax_merge(best, bi, v.y, base + 1);
            if (!(skip & 4u)) argmax_merge(best, bi, v.z, base + 2);
            if (!(skip & 8u)) argmax_merge(best, bi, v.w, base + 3);
            if (so) {
                if (!skip) {
                    *reinterpret_cast<float4*>(so + base) = v;
                } else {
                    if (!(skip & 1u)) so[base] = v.x;
                    if (!(skip & 2u)) so[base + 1] = v.y;
                    if (!(skip & 4u)) so[base + 2] = v.z;
                    if (!(skip & 8u)) so[base + 3] = v.w;
                }
            }
        }
        tail = beg + n4 * 4;
    }
    for (int t = tail + threadIdx.x; t < end; t += blockDim.x) {
        if ((ovr[(t - beg) >> 5] >> ((t - beg) & 31)) & 1u) continue;
        const float v = forced ? -INFINITY : (has_static ? p[t] + __ldg(static_add + t) : p[t]);
        argmax_merge(best, bi, v, t);
        if (so) so[t] = v;
    }
    // listed tokens: a token listed more than once resolves to the same value from every entry
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
        const int2 en = ent[e];
        const int t = en.x & 0x3fffffff;
        if (t < beg || t >= end) continue;
        const int kind = static_cast<int>(static_cast<unsigned>(en.x) >> 30);
        float v;
        if (kind == LP_SET) {
            v = __int_as_float(en.y);
        } else if (kind == LP_MASK || ((msk[(t - beg) >> 5] >> ((t - beg) & 31)) & 1u)) {
            v = -INFINITY;
        } else {   // LP_ADD: a token masked in static_add stays masked whatever its sequence bias
            const float s = has_static ? __ldg(static_add + t) : 0.f;
            v = (s == -INFINITY) ? -INFINITY : p[t] + __int_as_float(en.y);
        }
        argmax_merge(best, bi, v, t);
        if (so) so[t] = v;
    }
    __shared__ float sb[8];
    __shared__ int si[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) argmax_merge(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
    if ((threadIdx.x & 31) == 0) {
        sb[threadIdx.x >> 5] = best;
        si[threadIdx.x >> 5] = bi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) argmax_merge(best, bi, sb[w], si[w]);
        pmax[row * AM_SPLIT + sp] = best;
        pidx[row * AM_SPLIT + sp] = bi;
        trace_mark(trace, 3);
    }
}

size_t logits_process_scratch_bytes(int B, int cap) {
    return argmax_scratch_bytes(B) + static_cast<size_t>(B) * (static_cast<size_t>(cap) + 1) * sizeof(int2);
}

int logits_process_argmax(cudaStream_t stream, const float* logits, int B, int V, const int64_t* prompt, const int64_t* generated, int ld,
                          const int* gen_idx, const int* tables, const float* static_add, int cap, float* scores, int64_t* out,
                          void* scratch) {
    if (B <= 0) return 0;
    AF3_REQUIRE(logits && prompt && generated && gen_idx && tables && static_add && out && scratch, "logits_process_argmax: null argument");
    AF3_REQUIRE(cap >= 1 && ld >= 1, "logits_process_argmax: cap and ld must be positive");
    AF3_REQUIRE(V >= 1 && ((V + AM_SPLIT - 1) / AM_SPLIT + 3) / 4 * 4 <= LP_MAXW * 32, "logits_process_argmax: V too large");
    float* pmax = static_cast<float*>(scratch);
    int* pidx = reinterpret_cast<int*>(pmax + static_cast<size_t>(B) * AM_SPLIT);
    int2* row_info = reinterpret_cast<int2*>(static_cast<char*>(scratch) + argmax_scratch_bytes(B));
    int2* list = row_info + B;
    AF3_CHECK_CUDA(launch_kernel(logits_rules_kernel, dim3(B), dim3(256), 0, stream, prompt, generated, ld, V, gen_idx, tables, list, row_info,
                                 cap, trace_next_slot()));
    AF3_CHECK_CUDA(launch_kernel(logits_process_partial_kernel, dim3(B, AM_SPLIT), dim3(256), 0, stream, logits, V, static_add, tables,
                                 static_cast<const int2*>(list), static_cast<const int2*>(row_info), cap, scores, pmax, pidx,
                                 trace_next_slot()));
    AF3_CHECK_CUDA(launch_kernel(argmax_final_kernel, dim3(B), dim3(32), 0, stream, static_cast<const float*>(pmax),
                                 static_cast<const int*>(pidx), out, trace_next_slot()));
    return 0;
}

}  // namespace af3
