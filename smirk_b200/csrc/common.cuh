// Shared helpers for the smirk_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <string>
#include <vector>
#include "../../include/smirk_b200.h"

namespace smk {

void set_error(const char* fmt, ...);

#define SMK_CHECK_CUDA(expr)                                                            \
    do {                                                                                \
        cudaError_t _e = (expr);                                                        \
        if (_e != cudaSuccess) {                                                        \
            smk::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return (int)_e;                                                             \
        }                                                                               \
    } while (0)

#define SMK_REQUIRE(cond, ...)                                                          \
    do {                                                                                \
        if (!(cond)) { smk::set_error(__VA_ARGS__); return -1; }                        \
    } while (0)

// Launch bookkeeping: every kernel launch site calls SMK_TAG(...) first.  It counts launches (the
// `gpu_launches` figure bench.py reports) and, when the built-in profiler is enabled
// (smk_profiler_enable), brackets the launch with CUDA events on the launching stream so bench.py can
// report per-kernel time, algorithmic bytes and FLOPs without an external profiler.
void prof_begin(const char* tag, double bytes, double flops, cudaStream_t st);
void prof_end();
extern bool g_prof_detail;
bool profiling();                      // true while the event profiler is on (callers then serialise side streams)
const char* prof_shape_tag(const char* base, long m, long k, long n);   // interned "base:M.._K.._N.."
#define SMK_TAG(tag, bytes, flops, st) smk::prof_begin(tag, (double)(bytes), (double)(flops), st)
#define SMK_CHECK_LAUNCH() do { smk::prof_end(); SMK_CHECK_CUDA(cudaGetLastError()); } while (0)

// Device buffers owned by a handle (constants only; forwards never allocate).
struct DeviceArena {
    std::vector<void*> ptrs;
    ~DeviceArena() { for (void* p : ptrs) cudaFree(p); }
    template <typename T>
    cudaError_t upload(const T* host, size_t n, T** out) {
        void* d = nullptr;
        cudaError_t e = cudaMalloc(&d, n * sizeof(T) + 16);
        if (e != cudaSuccess) return e;
        ptrs.push_back(d);
        e = cudaMemcpy(d, host, n * sizeof(T), cudaMemcpyHostToDevice);
        *out = (T*)d;
        return e;
    }
    template <typename T>
    cudaError_t upload(const std::vector<T>& v, T** out) { return upload(v.data(), v.size(), out); }
    template <typename T>
    cudaError_t alloc(size_t n, T** out) {                  // unset: a live handle's weights, written on the device
        void* d = nullptr;
        cudaError_t e = cudaMalloc(&d, n * sizeof(T) + 16);
        if (e != cudaSuccess) return e;
        ptrs.push_back(d);
        *out = (T*)d;
        return e;
    }
};

// Bump allocator over the caller-provided workspace (256-byte aligned slices).
struct Workspace {
    char* base; size_t size; size_t off = 0;
    Workspace(void* p, size_t n) : base((char*)p), size(n) {}
    template <typename T> T* take(size_t n) {
        size_t bytes = (n * sizeof(T) + 255) & ~size_t(255);
        if (off + bytes > size) return nullptr;
        T* r = (T*)(base + off); off += bytes; return r;
    }
};
static inline size_t ws_round(size_t bytes) { return (bytes + 255) & ~size_t(255); }

// Walks the host tensor list of a create call (state_dict order); null past the end.
struct TensorCursor {
    const float* const* t; int n; int i = 0;
    const float* next() { return i < n ? t[i++] : nullptr; }
};

// Eval-mode BatchNorm folded into a per-channel scale and bias: s = g / sqrt(var + eps), b' = beta - mu * s.
static inline void fold_bn(const float* g, const float* beta, const float* mu, const float* var, int n, float eps, float* s, float* b) {
    for (int o = 0; o < n; ++o) {
        const float so = g[o] / sqrtf(var[o] + eps);
        s[o] = so; b[o] = beta[o] - mu[o] * so;
    }
}

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// Streaming multiprocessors of the current device (cached per device ordinal): the size of a persistent grid.
int num_sms();

// Blocks of 256 threads for a grid-stride loop over `total` items: one item per thread, at most 16 blocks per SM.
static inline int grid_of(long total) { return (int)std::min<long>((total + 255) / 256, 16L * num_sms()); }

// TF-SAME padding of a 3x3 window: zero rows / columns before the first input pixel (TensorFlow pads the odd one after).
static inline int same_pad_begin(int H, int stride) {
    const int out = (H + stride - 1) / stride;
    return std::max((out - 1) * stride + 3 - H, 0) / 2;
}

// Where a grad-mode forward keeps the activations its backward needs: named [B,H,W,C] fp32 tensors in one caller-owned
// buffer, in the order they were added.  A tensor's offset is B times its per-image offset, and every tensor starts on a
// 64-float boundary so float4 / TMA access to it stays aligned whatever B is.
struct SavedLayout {
    std::vector<std::string> name;
    std::vector<size_t> off;           // per-image float offset of each tensor
    std::vector<int> hwc;              // H, W, C of each tensor
    size_t total = 0;                  // floats per image

    int add(const std::string& n, int H, int W, int C) {      // -> the tensor's index
        name.push_back(n); off.push_back(total); hwc.insert(hwc.end(), {H, W, C});
        total += ((size_t)H * W * C + 63) / 64 * 64;
        return (int)name.size() - 1;
    }
    size_t bytes(int B) const { return B > 0 ? total * (size_t)B * sizeof(float) : 0; }
};

// The `smk_*_saved_tensor` query of a handle's layout L (null for a null handle); fn names the entry point in errors.
static inline int saved_tensor(const SavedLayout* L, const char* fn, int B, int i, const char** name, size_t* offset, int* dims) {
    SMK_REQUIRE(L && name && offset && dims, "%s: null argument", fn);
    SMK_REQUIRE(B >= 0, "%s: negative batch", fn);
    SMK_REQUIRE(i >= 0 && i < (int)L->name.size(), "%s: index %d out of range (%d tensors)", fn, i, (int)L->name.size());
    *name = L->name[i].c_str();
    *offset = L->off[i] * (size_t)B;
    dims[0] = B; dims[1] = L->hwc[3 * i]; dims[2] = L->hwc[3 * i + 1]; dims[3] = L->hwc[3 * i + 2];
    return 0;
}

#ifdef __CUDACC__
// Launch errors surface through cudaGetLastError in SMK_CHECK_LAUNCH.
#define SMK_LAUNCH(kernel, grid, block, smem, st, ...) kernel<<<grid, block, smem, st>>>(__VA_ARGS__)

// cudaFuncAttributeMaxDynamicSharedMemorySize is per device and per function: set it the first time Kernel is
// launched on a device.  One bit per device ordinal (ordinals >= 64 set it on every call).
template <auto Kernel>
cudaError_t set_max_dynamic_smem(int bytes) {
    static unsigned long long configured_mask = 0;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const unsigned long long bit = dev < 64 ? 1ull << dev : 0;
    if (bit && (__atomic_load_n(&configured_mask, __ATOMIC_RELAXED) & bit)) return cudaSuccess;
    e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) __atomic_fetch_or(&configured_mask, bit, __ATOMIC_RELAXED);
    return e;
}
#endif

// TF32 rounding (round-to-nearest, ties away: PTX cvt.rna).  The tensor cores read fp32 words from shared
// memory and simply ignore the 13 low mantissa bits (truncation, a systematic bias); operands that feed
// a tensor-core layer are therefore rounded once, where they are produced: weights on the host at pack
// time, activations in the epilogue of the kernel that writes them — what cuDNN/CUTLASS TF32 kernels
// do with cvt.rna in registers before mma.
#ifdef __CUDACC__
__device__ __forceinline__ float round_tf32(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
// float4 fused multiply-adds (four IEEE fmaf each) of the CUDA-core inner loops.
__device__ __forceinline__ void fma4_acc(float4& acc, const float4& x, const float4& k) {    // acc += x * k
    acc.x = fmaf(x.x, k.x, acc.x); acc.y = fmaf(x.y, k.y, acc.y); acc.z = fmaf(x.z, k.z, acc.z); acc.w = fmaf(x.w, k.w, acc.w);
}
__device__ __forceinline__ void fma4_s(float4& acc, float x, const float4& k) {              // acc += x * k (scalar x)
    acc.x = fmaf(x, k.x, acc.x); acc.y = fmaf(x, k.y, acc.y); acc.z = fmaf(x, k.z, acc.z); acc.w = fmaf(x, k.w, acc.w);
}
__device__ __forceinline__ float4 fma4(const float4& x, const float4& s, const float4& b) {  // x * s + b
    return make_float4(fmaf(x.x, s.x, b.x), fmaf(x.y, s.y, b.y), fmaf(x.z, s.z, b.z), fmaf(x.w, s.w, b.w));
}
#endif
static inline float round_tf32_host(float x) {
    uint32_t u; memcpy(&u, &x, 4);
    if ((u & 0x7F800000u) == 0x7F800000u) return x;          // inf / nan
    u = (u + 0x1000u) & 0xFFFFE000u;
    float r; memcpy(&r, &u, 4); return r;
}

}  // namespace smk
