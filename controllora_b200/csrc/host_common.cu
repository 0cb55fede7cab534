#include "host_common.h"

#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <string>
#include <unordered_map>

namespace clb {

static thread_local char g_err[1024] = "";
static std::atomic<long long> g_launches{0};

int set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int num_sms() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (sms <= 0) sms = 132;
    }
    return sms;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

static std::mutex g_tm_mutex;
static std::unordered_map<std::string, CUtensorMap> g_tm_cache;

int get_tensor_map(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, int swizzle_bytes) {
    if (rank < 1 || rank > 5) return set_error(CL_ERR_INVALID, "tensor map rank %d", rank);
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0) return set_error(CL_ERR_INVALID, "tensor map base not 16B aligned");
    struct Key {
        const void* ptr;
        int rank, sw;
        uint64_t dims[5], strides[4];
        uint32_t box[5];
    } key;
    memset(&key, 0, sizeof(key));
    key.ptr = ptr; key.rank = rank; key.sw = swizzle_bytes;
    for (int i = 0; i < rank; ++i) { key.dims[i] = dims[i]; key.box[i] = box[i]; }
    for (int i = 0; i + 1 < rank; ++i) {
        key.strides[i] = strides_bytes[i];
        if (strides_bytes[i] % 16 != 0) return set_error(CL_ERR_INVALID, "tensor map stride %d not a multiple of 16 B", i);
    }
    std::string k(reinterpret_cast<const char*>(&key), sizeof(key));
    std::lock_guard<std::mutex> lock(g_tm_mutex);
    auto it = g_tm_cache.find(k);
    if (it != g_tm_cache.end()) {
        *out = it->second;
        return CL_OK;
    }
    EncodeTiledFn fn = get_encode_fn();
    if (fn == nullptr) return set_error(CL_ERR_CUDA, "cuTensorMapEncodeTiled entry point not found (no CUDA driver?)");
    cuuint64_t gdims[5];
    cuuint64_t gstr[4];
    cuuint32_t gbox[5], estr[5];
    for (int i = 0; i < rank; ++i) { gdims[i] = dims[i]; gbox[i] = box[i]; estr[i] = 1; }
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), gdims, gstr, gbox,
                    estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE),
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        return set_error(CL_ERR_CUDA,
                         "cuTensorMapEncodeTiled failed (%d): rank %d dims %llu %llu %llu %llu %llu box %u %u %u %u %u",
                         (int)r, rank, (unsigned long long)key.dims[0], (unsigned long long)key.dims[1],
                         (unsigned long long)key.dims[2], (unsigned long long)key.dims[3],
                         (unsigned long long)key.dims[4], key.box[0], key.box[1], key.box[2], key.box[3], key.box[4]);
    }
    if (g_tm_cache.size() > 200000) g_tm_cache.clear();
    g_tm_cache.emplace(std::move(k), *out);
    return CL_OK;
}

}  // namespace clb

extern "C" const char* cl_last_error(void) { return clb::g_err; }
extern "C" int cl_version(void) { return 101; }
extern "C" int64_t cl_launch_count(void) { return clb::g_launches.load(); }
