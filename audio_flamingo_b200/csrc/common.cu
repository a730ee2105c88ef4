#include "common.h"

#include <mutex>

namespace af3 {

static thread_local std::string g_last_error;

void set_last_error(const std::string& msg) { g_last_error = msg; }
int fail(const std::string& msg) {
    g_last_error = msg;
    return 1;
}
const char* last_error_cstr() { return g_last_error.c_str(); }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
        if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<PFN_encodeTiled>(p);
    });
    return fn;
}

static int encode(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_b,
                  const cuuint32_t* box, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,
                  CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
    PFN_encodeTiled fn = get_encode();
    if (!fn) return fail("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = fn(map, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_b,
                    box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        return fail("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r) + " (rank " +
                    std::to_string(rank) + ", dims " + std::to_string(dims[0]) + "x" + std::to_string(dims[1]) +
                    ", box " + std::to_string(box[0]) + "x" + std::to_string(box[1]) + ")");
    }
    return 0;
}

int make_tmap_2d(CUtensorMap* map, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_elems,
                 uint32_t box_cols, uint32_t box_rows) {
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return fail("TMA base pointer must be 16-byte aligned");
    if ((pitch_elems * 2) % 16 != 0) return fail("TMA row pitch must be a multiple of 16 bytes");
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {pitch_elems * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    return encode(map, base, 2, dims, strides, box);
}

int make_tmap_2d_u8(CUtensorMap* map, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch_bytes, uint32_t box_cols,
                    uint32_t box_rows, bool swizzle_64b) {
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return fail("TMA base pointer must be 16-byte aligned");
    if (pitch_bytes % 16 != 0) return fail("TMA row pitch must be a multiple of 16 bytes");
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {pitch_bytes};
    cuuint32_t box[2] = {box_cols, box_rows};
    return encode(map, base, 2, dims, strides, box, CU_TENSOR_MAP_DATA_TYPE_UINT8,
                  swizzle_64b ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B);
}

int make_tmap_3d(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t p1_elems,
                 uint64_t p2_elems, uint32_t box0, uint32_t box1, uint32_t box2) {
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return fail("TMA base pointer must be 16-byte aligned");
    if ((p1_elems * 2) % 16 != 0 || (p2_elems * 2) % 16 != 0) return fail("TMA pitches must be multiples of 16 bytes");
    cuuint64_t dims[3] = {d0, d1, d2};
    cuuint64_t strides[2] = {p1_elems * 2, p2_elems * 2};
    cuuint32_t box[3] = {box0, box1, box2};
    return encode(map, base, 3, dims, strides, box);
}

static bool g_pdl = false;
bool pdl_enabled() { return g_pdl; }
void set_pdl(bool on) { g_pdl = on; }

// ---- in-graph timeline (see common.h)
static unsigned long long* g_trace_buf = nullptr;
static size_t g_trace_slots = 0;
static int g_trace_seq = 0;
int trace_begin(void* buf, size_t bytes) {
    g_trace_buf = static_cast<unsigned long long*>(buf);
    g_trace_slots = bytes / (sizeof(unsigned long long) * TRACE_CTAS * TRACE_MARKS);
    g_trace_seq = 0;
    return 0;
}
int trace_end() {
    const int n = g_trace_seq;
    g_trace_buf = nullptr;
    g_trace_slots = 0;
    return n;
}
int trace_seq() { return g_trace_seq; }
unsigned long long* trace_next_slot() {
    if (!g_trace_buf) return nullptr;
    if (static_cast<size_t>(g_trace_seq) >= g_trace_slots) {
        ++g_trace_seq;  // counted, not recorded
        return nullptr;
    }
    return g_trace_buf + static_cast<size_t>(g_trace_seq++) * TRACE_CTAS * TRACE_MARKS;
}

int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return dev;
}

int sm_count() {
    static int n[128] = {0};
    const int dev = current_device() & 127;
    if (n[dev] == 0) {
        cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
        if (n[dev] <= 0) n[dev] = 132;
    }
    return n[dev];
}

}  // namespace af3
