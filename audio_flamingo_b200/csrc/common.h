// Host-side helpers shared by all translation units of libaf3b200.so:
// error reporting for the C ABI, TMA tensor-map construction (driver entry point fetched at run time so the
// library links against cudart only), and device properties.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

namespace af3 {

typedef __nv_bfloat16 bf16;

void set_last_error(const std::string& msg);
int fail(const std::string& msg);  // records msg, returns a non-zero status

#define AF3_CHECK_CUDA(expr)                                                                        \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess)                                                                      \
            return af3::fail(std::string(#expr) + " -> " + cudaGetErrorString(_e) + " @" + __FILE__ + \
                             ":" + std::to_string(__LINE__));                                       \
    } while (0)

#define AF3_CHECK_LAUNCH() AF3_CHECK_CUDA(cudaGetLastError())

#define AF3_REQUIRE(cond, msg)                                          \
    do {                                                                \
        if (!(cond)) return af3::fail(std::string("af3: ") + (msg));    \
    } while (0)

// bf16 row-major tensor maps with 128-byte swizzle; box inner extent is always 64 elements (128 B).
// 2-D: dims (inner = cols, outer = rows), row pitch in elements.
int make_tmap_2d(CUtensorMap* map, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_elems,
                 uint32_t box_cols, uint32_t box_rows);
// The same for one-byte elements (e4m3): box inner extent 128 elements (128 B), pitch in bytes.  swizzle_64b: 64-byte swizzle
// for a 64-byte box inner extent (packed int4 weights, two nibbles per byte).
int make_tmap_2d_u8(CUtensorMap* map, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_bytes, uint32_t box_cols,
                    uint32_t box_rows, bool swizzle_64b = false);
// 3-D: dims (d0 = cols, d1, d2) with element pitches p1, p2.
int make_tmap_3d(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t p1_elems,
                 uint64_t p2_elems, uint32_t box0, uint32_t box1, uint32_t box2);

int sm_count();        // of the CURRENT device (cached per device ordinal)
int current_device();

// One-time per-DEVICE kernel setup (cudaFuncSetAttribute is per device): a model on cuda:1 after one on cuda:0 in the
// same process must configure its kernels again (ADVICE r01).  Usage: static DeviceOnce once; if (once.first()) {...}
struct DeviceOnce {
    unsigned long long mask[2] = {0, 0};  // device ordinals 0..127
    bool first() {
        const int d = current_device() & 127;
        const unsigned long long bit = 1ull << (d & 63);
        if (mask[d >> 6] & bit) return false;
        mask[d >> 6] |= bit;
        return true;
    }
};

// Programmatic dependent launch for the decode-step kernel chain (af3_set_pdl).  launch_kernel() adds the
// cudaLaunchAttributeProgrammaticStreamSerialization attribute when enabled; every kernel launched through it calls
// pdl_wait() before touching data produced by earlier kernels.
bool pdl_enabled();
void set_pdl(bool on);

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// In-graph timeline of the decode-step kernel chain (af3_trace_begin / af3_trace_end, profiles/decode_timeline.py).
// While a trace is open every launch of an instrumented kernel gets the next slot of TRACE_CTAS x TRACE_MARKS
// %globaltimer stamps in the caller's device buffer (the slot address is baked into the launch, so a captured CUDA
// graph keeps writing the same slots on every replay: the buffer then holds the timeline of the LAST replay, with
// programmatic dependent launch on and nothing serialised -- what ncu cannot show).  nullptr = tracing off.
constexpr int TRACE_CTAS = 160;   // CTAs recorded per launch (linear block index below this)
constexpr int TRACE_MARKS = 4;    // 0 entry, 1 after griddepcontrol.wait, 2 main loop done, 3 exit
unsigned long long* trace_next_slot();

}  // namespace af3
