// Peer-mapped gather buffers: the multi-GPU all-gather of the final outputs (SURVEY.md 8e; the reference itself has no
// multi-GPU code) done with copy-engine pushes over NVLink instead of a collective kernel.
//
// Why not only NCCL: the compute kernels of this library are persistent (one CTA per SM striding over their work items).
// A collective kernel that occupies a few SMs while they run turns every concurrent persistent launch into two waves.  A push
// from the copy engines takes no SM: each rank owns one gather buffer [world][shard], maps every peer's buffer through CUDA
// IPC once, and after each batch copies its packed shard into slot `rank` of every peer's buffer on a communication stream.
#include "common.cuh"
#include <cstring>
#include <vector>

extern "C" int smk_peer_alloc(size_t bytes, void** ptr, unsigned char* handle64) {
    SMK_REQUIRE(ptr && handle64 && bytes > 0, "smk_peer_alloc: null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
    void* p = nullptr;
    SMK_CHECK_CUDA(cudaMalloc(&p, bytes));           // set-up time only; a plain (not pooled) allocation so the handle's base is `p`
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) { cudaFree(p); SMK_CHECK_CUDA(e); }
    memcpy(handle64, &h, 64);
    *ptr = p;
    return 0;
}

extern "C" int smk_peer_free(void* ptr) {
    if (ptr) SMK_CHECK_CUDA(cudaFree(ptr));
    return 0;
}

// Maps another process's buffer (same node) into this process's current device context; peer access is enabled on demand.
extern "C" int smk_peer_open(const unsigned char* handle64, void** ptr) {
    SMK_REQUIRE(ptr && handle64, "smk_peer_open: null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    SMK_CHECK_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return 0;
}

extern "C" int smk_peer_close(void* ptr) {
    if (ptr) SMK_CHECK_CUDA(cudaIpcCloseMemHandle(ptr));
    return 0;
}

// One copy per destination, spread over the fan's own streams so that several copy engines (and NVLink ports) work at once:
// on one stream the pushes to all peers would run one after another.  Ordered after the work already on `stream`; `stream` continues only after every copy (device-side waits).
struct SmkPeerFan {
    std::vector<cudaStream_t> streams;
    std::vector<cudaEvent_t> done;
    cudaEvent_t ready = nullptr;
};

extern "C" int smk_peer_fan_create(int n_streams, SmkPeerFan** out) {
    SMK_REQUIRE(out && n_streams >= 1 && n_streams <= 16, "smk_peer_fan_create: 1..16 streams");
    SmkPeerFan* f = new SmkPeerFan();
    cudaError_t e = cudaEventCreateWithFlags(&f->ready, cudaEventDisableTiming);
    for (int i = 0; i < n_streams && e == cudaSuccess; ++i) {
        cudaStream_t s = nullptr; cudaEvent_t ev = nullptr;
        e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
        if (e == cudaSuccess) { f->streams.push_back(s); e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming); }
        if (e == cudaSuccess) f->done.push_back(ev);
    }
    if (e != cudaSuccess) {
        for (auto s : f->streams) cudaStreamDestroy(s);
        for (auto ev : f->done) cudaEventDestroy(ev);
        if (f->ready) cudaEventDestroy(f->ready);
        delete f;
        SMK_CHECK_CUDA(e);
    }
    *out = f;
    return 0;
}

extern "C" void smk_peer_fan_destroy(SmkPeerFan* f) {
    if (!f) return;
    for (auto s : f->streams) cudaStreamDestroy(s);
    for (auto ev : f->done) cudaEventDestroy(ev);
    if (f->ready) cudaEventDestroy(f->ready);
    delete f;
}

extern "C" int smk_peer_fan_push(SmkPeerFan* f, void* const* dsts, int n, const void* src, size_t bytes, void* stream) {
    SMK_REQUIRE(f && dsts && src && n >= 0, "smk_peer_fan_push: null argument");
    if (n == 0 || bytes == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const int ns = (int)f->streams.size(), used = n < ns ? n : ns;
    SMK_CHECK_CUDA(cudaEventRecord(f->ready, st));
    for (int i = 0; i < used; ++i) SMK_CHECK_CUDA(cudaStreamWaitEvent(f->streams[i], f->ready, 0));
    for (int i = 0; i < n; ++i) {
        SMK_REQUIRE(dsts[i], "smk_peer_fan_push: null destination %d", i);
        SMK_CHECK_CUDA(cudaMemcpyAsync(dsts[i], src, bytes, cudaMemcpyDeviceToDevice, f->streams[i % ns]));
    }
    for (int i = 0; i < used; ++i) {
        SMK_CHECK_CUDA(cudaEventRecord(f->done[i], f->streams[i]));
        SMK_CHECK_CUDA(cudaStreamWaitEvent(st, f->done[i], 0));
    }
    return 0;
}

// dst may be local or peer-mapped; the copy runs on a copy engine, ordered on `stream`.
extern "C" int smk_peer_push(void* dst, const void* src, size_t bytes, void* stream) {
    SMK_REQUIRE(dst && src, "smk_peer_push: null pointer");
    if (bytes) SMK_CHECK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return 0;
}
