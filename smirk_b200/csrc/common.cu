// Error channel + version for the smirk_b200 C ABI.
#include "common.cuh"
#include <stdarg.h>

namespace smk {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// ---- launch counter + optional event profiler -------------------------------------------------------
struct ProfEntry { const char* tag; cudaEvent_t a, b; double bytes, flops; };
static std::vector<ProfEntry> g_entries;
static bool g_prof = false, g_pending = false;
static cudaStream_t g_pending_stream = nullptr;
static unsigned long long g_launches = 0;
bool g_prof_detail = false;          // level 2: GEMM / depthwise launches are tagged with their shape

const char* prof_shape_tag(const char* base, long m, long k, long n) {
    static std::vector<char*> pool;
    char buf[96];
    snprintf(buf, sizeof(buf), "%s:M%ld_K%ld_N%ld", base, m, k, n);
    for (char* p : pool) if (strcmp(p, buf) == 0) return p;
    pool.push_back(strdup(buf));
    return pool.back();
}

void prof_begin(const char* tag, double bytes, double flops, cudaStream_t st) {
    __atomic_add_fetch(&g_launches, 1ULL, __ATOMIC_RELAXED);
    if (!g_prof) return;
    ProfEntry e{tag, nullptr, nullptr, bytes, flops};
    if (cudaEventCreate(&e.a) != cudaSuccess || cudaEventCreate(&e.b) != cudaSuccess) return;
    cudaEventRecord(e.a, st);
    g_entries.push_back(e);
    g_pending = true; g_pending_stream = st;
}
bool profiling() { return g_prof; }
int num_sms() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
    if (dev < 64 && cached[dev]) return cached[dev];
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    if (dev < 64) cached[dev] = n;
    return n;
}
void prof_end() {
    if (!g_prof || !g_pending) return;
    cudaEventRecord(g_entries.back().b, g_pending_stream);
    g_pending = false;
}
}  // namespace smk

extern "C" unsigned long long smk_launch_count(void) { return smk::g_launches; }
extern "C" void smk_profiler_enable(int on) { smk::g_prof = on != 0; smk::g_prof_detail = on >= 2; }
extern "C" void smk_profiler_reset(void) {
    for (auto& e : smk::g_entries) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
    smk::g_entries.clear();
}
// Writes one line per kernel tag: "tag launches total_ms bytes flops\n" (bytes/flops summed over launches).
extern "C" int smk_profiler_report(char* buf, size_t n) {
    cudaDeviceSynchronize();
    struct Agg { const char* tag; long launches; double ms, bytes, flops; };
    std::vector<Agg> aggs;
    for (auto& e : smk::g_entries) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, e.a, e.b) != cudaSuccess) continue;
        Agg* a = nullptr;
        for (auto& x : aggs) if (strcmp(x.tag, e.tag) == 0) { a = &x; break; }
        if (!a) { aggs.push_back(Agg{e.tag, 0, 0, 0, 0}); a = &aggs.back(); }
        a->launches++; a->ms += ms; a->bytes += e.bytes; a->flops += e.flops;
    }
    size_t off = 0;
    for (auto& a : aggs) {
        int w = snprintf(buf + off, off < n ? n - off : 0, "%s %ld %.6f %.0f %.0f\n", a.tag, a.launches, a.ms, a.bytes, a.flops);
        if (w < 0 || off + (size_t)w >= n) return -1;
        off += (size_t)w;
    }
    if (off < n) buf[off] = 0;
    return (int)aggs.size();
}

extern "C" int smk_version(void) { return SMK_VERSION; }
extern "C" const char* smk_last_error(void) { return smk::g_err; }
