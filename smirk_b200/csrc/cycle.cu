// The cycle path's parameter augmentation (src/smirk_trainer.py:189-248) with its random draws made on the device
// (include/smirk_b200.h).  The reference draws a permutation on the host, loops over template rows in Python and
// issues ~30 small torch ops; here the whole augmentation of Ke*B rows is one single-CTA launch: both permutations
// (ranks of Philox keys in shared memory), every Bernoulli / normal / uniform and the template picks come from the
// counter-based generator of csrc/philox.cuh, and the arithmetic repeats the reference's fp32 ops one by one (explicit
// round-to-nearest intrinsics, no FMA contraction), so given the exported draws the result is bitwise the reference's.
#include "common.cuh"
#include "philox.cuh"
#include <math.h>
#include <vector>

namespace {

using smk::U4;
using smk::philox;
using smk::u01;

constexpr int kThreads = 1024;
constexpr int kMaxRows = 2048;           // Ke * B: the permutation tables live in shared memory (26 KB)

// one Philox stream id per kind of draw (the masking stage uses 0-3 on its own rng_state)
enum : uint32_t { kGids = 0, kPerm1, kMask, kNormA, kRow, kJaw, kEye, kPick };

struct CycleIO {
    const float* in[6];
    float* out[6];
    int dim[6];               // pose, cam, shape, expression, jaw, eyelid
};

__device__ __forceinline__ float clampf(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }   // NaN stays NaN

// N(0, 1) by Box-Muller from two uniforms
__device__ __forceinline__ float normal(uint32_t a, uint32_t b) {
    return sqrtf(-2.f * logf(1.f - u01(a))) * cosf(6.2831853f * u01(b));
}

// an unbiased-enough index in [0, n): the high word of r * n (bias < n / 2^32)
__device__ __forceinline__ int below(uint32_t r, int n) { return (int)(((uint64_t)r * (uint64_t)n) >> 32); }

// perm = a uniformly random permutation of [0, n): ranks of (32-bit Philox key, index) pairs, which are distinct.
__device__ void random_perm(uint64_t seed, uint64_t ctr, uint32_t stream, int n, int* perm, uint32_t* keys) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) keys[i] = philox(seed, ctr, stream, 0u, (uint32_t)i).x;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t k = keys[i];
        int rank = 0;
        for (int j = 0; j < n; ++j) { const uint32_t q = keys[j]; rank += (q < k) || (q == k && j < i); }
        perm[rank] = i;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kThreads)
cycle_augment_kernel(CycleIO io, int B, int R, int use_eyelids, const float* __restrict__ tmpl, const int* __restrict__ tmpl_off, int n_keys,
                     int n_exp, uint64_t* __restrict__ rng, SmkCycleDraws dbg) {
    __shared__ int gids[kMaxRows], pos[kMaxRows];
    __shared__ int perm1[kMaxRows / 4 + 1];
    __shared__ uint32_t keys[kMaxRows];
    const uint64_t seed = rng[0], ctr = rng[1];
    // smirk_trainer.py:200-202: gids = randperm(R), split at R/4, 2R/4, 3R/4
    const int c1 = R / 4, c2 = 2 * R / 4, c3 = 3 * R / 4;
    random_perm(seed, ctr, kGids, R, gids, keys);
    for (int i = threadIdx.x; i < R; i += blockDim.x) pos[gids[i]] = i;
    const int m1 = c2 - c1;
    random_perm(seed, ctr, kPerm1, m1, perm1, keys);   // :215 the in-group permutation of group 1 (syncs)
    if (dbg.gids) for (int i = threadIdx.x; i < R; i += blockDim.x) dbg.gids[i] = gids[i];
    if (dbg.perm1) for (int i = threadIdx.x; i < m1; i += blockDim.x) dbg.perm1[i] = perm1[i];

    const int E = io.dim[3];
    // ---- expression (:206-223, :238-239); group g's row k is output row gids[start_g + k] ----
    for (int idx = threadIdx.x; idx < R * E; idx += blockDim.x) {
        const int r = idx / E, e = idx - r * E, p = pos[r];
        const float x = io.in[3][(size_t)(r % B) * E + e];
        const U4 rr = philox(seed, ctr, kRow, 0u, (uint32_t)p);                 // per-row uniforms (indexed by position)
        const U4 na = philox(seed, ctr, kNormA, (uint32_t)p, (uint32_t)e);
        float v;
        if (p < c1) {                                   // 1 of 4: random expressions
            const int k = p;
            const float pm = u01(philox(seed, ctr, kMask, (uint32_t)p, (uint32_t)e).x) < 0.5f ? 1.f : 0.f;
            const float a = normal(na.x, na.y), bn = normal(na.z, na.w);
            const float ua = u01(rr.x), ub = u01(rr.y);
            const float nw = __fadd_rn(__fmul_rn(__fmul_rn(a, __fadd_rn(1.f, __fmul_rn(2.f, ua))), pm), x);
            v = __fadd_rn(clampf(nw, -4.f, 4.f), __fmul_rn(__fadd_rn(0.f, __fmul_rn(0.2f, ub)), bn));
            if (dbg.param_mask) dbg.param_mask[(size_t)k * E + e] = pm;
            if (dbg.randn0a) dbg.randn0a[(size_t)k * E + e] = a;
            if (dbg.randn0b) dbg.randn0b[(size_t)k * E + e] = bn;
            if (e == 0 && dbg.rand0a) dbg.rand0a[k] = ua;
            if (e == 0 && dbg.rand0b) dbg.rand0b[k] = ub;
        } else if (p < c2) {                            // 2 of 4: permutation of the group's expressions
            const int k = p - c1;
            const float xp = io.in[3][(size_t)(gids[c1 + perm1[k]] % B) * E + e];
            const float n = normal(na.x, na.y), ua = u01(rr.x), ub = u01(rr.y);
            v = __fadd_rn(__fmul_rn(__fadd_rn(0.25f, __fmul_rn(1.25f, ua)), xp), __fmul_rn(__fadd_rn(0.f, __fmul_rn(0.2f, ub)), n));
            if (dbg.randn1) dbg.randn1[(size_t)k * E + e] = n;
            if (e == 0 && dbg.rand1a) dbg.rand1a[k] = ua;
            if (e == 0 && dbg.rand1b) dbg.rand1b[k] = ub;
        } else if (p < c3) {                            // 3 of 4: template injection (a key uniformly, then a row of it)
            const int k = p - c2;
            const U4 pk = philox(seed, ctr, kPick, 0u, (uint32_t)k);
            const int key = below(pk.x, n_keys), row = below(pk.y, tmpl_off[key + 1] - tmpl_off[key]);
            const float n = normal(na.x, na.y), ua = u01(rr.x), ub = u01(rr.y);
            const float t = e < n_exp ? __fmul_rn(__fadd_rn(0.25f, __fmul_rn(1.25f, ua)), tmpl[(size_t)(tmpl_off[key] + row) * n_exp + e]) : x;
            v = __fadd_rn(t, __fmul_rn(__fadd_rn(0.f, __fmul_rn(0.2f, ub)), n));
            if (dbg.randn2) dbg.randn2[(size_t)k * E + e] = n;
            if (e == 0 && dbg.rand2a) dbg.rand2a[k] = ua;
            if (e == 0 && dbg.rand2b) dbg.rand2b[k] = ub;
            if (e == 0 && dbg.tmpl_key) dbg.tmpl_key[k] = key;
            if (e == 0 && dbg.tmpl_row) dbg.tmpl_row[k] = row;
        } else {                                        // 4 of 4: zero expression (x * 0 keeps the sign of zero)
            const int k = p - c3;
            const float n = normal(na.x, na.y), u = u01(rr.x);
            v = __fadd_rn(__fmul_rn(x, 0.0f), __fmul_rn(__fadd_rn(0.f, __fmul_rn(0.2f, u)), n));
            if (dbg.randn3) dbg.randn3[(size_t)k * E + e] = n;
            if (e == 0 && dbg.rand3) dbg.rand3[k] = u;
        }
        io.out[3][(size_t)r * E + e] = v;
    }
    // ---- jaw (:226-228, :241): + randn * 0.2 * ([1, .1, .1] * Bernoulli(0.5)), jaw[:, 0] clamped to [0, 0.5] ----
    for (int idx = threadIdx.x; idx < R * 3; idx += blockDim.x) {
        const int r = idx / 3, j = idx - r * 3, p = pos[r];
        const float bm = u01(philox(seed, ctr, kJaw, 1u, (uint32_t)r).x) < 0.5f ? 1.f : 0.f;
        const U4 nj = philox(seed, ctr, kJaw, 0u, (uint32_t)idx);
        const float n = normal(nj.x, nj.y);
        const float s = __fmul_rn(j == 0 ? 1.f : 0.1f, bm);
        float v = __fadd_rn(io.in[4][(size_t)(r % B) * 3 + j], __fmul_rn(__fmul_rn(n, 0.2f), s));
        if (j == 0) v = clampf(v, 0.f, 0.5f);
        if (p >= c3) v = __fmul_rn(v, 0.0f);
        io.out[4][idx] = v;
        if (j == 0 && dbg.jaw_mask) dbg.jaw_mask[r] = bm;
        if (dbg.randn_jaw) dbg.randn_jaw[idx] = n;
    }
    // ---- eyelids (:231-233, :242): (-1 + 2U) * 0.25 and clamp to [0, 1] with use_eyelids; U(0,1) in group 4 always ----
    const int De = io.dim[5];
    for (int idx = threadIdx.x; idx < R * De; idx += blockDim.x) {
        const int r = idx / De, j = idx - r * De, p = pos[r];
        float v = io.in[5][(size_t)(r % B) * De + j];
        if (use_eyelids) {
            const float u = u01(philox(seed, ctr, kEye, 0u, (uint32_t)idx).x);
            v = clampf(__fadd_rn(v, __fmul_rn(__fadd_rn(-1.f, __fmul_rn(2.f, u)), 0.25f)), 0.f, 1.f);
            if (dbg.rand_eyelid) dbg.rand_eyelid[idx] = u;
        }
        if (p >= c3) {
            const int k = p - c3;
            v = u01(philox(seed, ctr, kEye, 1u, (uint32_t)(k * De + j)).x);
            if (dbg.rand3_eyelid) dbg.rand3_eyelid[(size_t)k * De + j] = v;
        }
        io.out[5][idx] = v;
    }
    // ---- pose, cam, shape: row r mod B (torch.cat(Ke * [v])) ----
    for (int t = 0; t < 3; ++t) {
        const int D = io.dim[t];
        for (int idx = threadIdx.x; idx < R * D; idx += blockDim.x) {
            const int r = idx / D;
            io.out[t][idx] = io.in[t][(size_t)(r % B) * D + (idx - r * D)];
        }
    }
    __syncthreads();                                    // every thread has read the counter: advance it
    if (threadIdx.x == 0) rng[1] = ctr + 1;
}

}  // namespace

struct SmkCycle {
    int n_keys, n_exp;
    float* rows;
    int* offsets;
    smk::DeviceArena arena;
};

extern "C" int smk_cycle_create(const SmkCycleDesc* desc, SmkCycle** out) {
    SMK_REQUIRE(desc && out && desc->row_offset && desc->rows, "smk_cycle_create: null argument");
    SMK_REQUIRE(desc->n_keys > 0 && desc->n_exp > 0, "smk_cycle_create: need at least one template key and n_exp > 0");
    SMK_REQUIRE(desc->row_offset[0] == 0, "smk_cycle_create: row_offset[0] must be 0");
    for (int k = 0; k < desc->n_keys; ++k)
        SMK_REQUIRE(desc->row_offset[k + 1] > desc->row_offset[k], "smk_cycle_create: template key %d has no rows", k);
    SmkCycle* h = new SmkCycle();
    h->n_keys = desc->n_keys; h->n_exp = desc->n_exp;
    const size_t total = (size_t)desc->row_offset[desc->n_keys];
    cudaError_t e = h->arena.upload(desc->rows, total * desc->n_exp, &h->rows);
    if (e == cudaSuccess) e = h->arena.upload(reinterpret_cast<const int*>(desc->row_offset), (size_t)desc->n_keys + 1, &h->offsets);
    if (e != cudaSuccess) { smk::set_error("smk_cycle_create: upload failed: %s", cudaGetErrorString(e)); delete h; return (int)e; }
    *out = h;
    return 0;
}

extern "C" void smk_cycle_destroy(SmkCycle* h) { delete h; }

extern "C" int smk_cycle_augment(const SmkCycle* h, const float* const* in, float* const* out, const int* dims, int B, int Ke, int use_eyelids,
                                 uint64_t* rng_state, const SmkCycleDraws* dbg, void* stream) {
    SMK_REQUIRE(h && in && out && dims && rng_state, "smk_cycle_augment: null argument");
    SMK_REQUIRE(B >= 1 && Ke >= 1 && (long)B * Ke <= kMaxRows, "smk_cycle_augment: need 1 <= B, 1 <= Ke and Ke * B <= %d", kMaxRows);
    CycleIO io;
    for (int t = 0; t < 6; ++t) {
        SMK_REQUIRE(in[t] && out[t] && dims[t] > 0, "smk_cycle_augment: tensor %d missing or empty", t);
        io.in[t] = in[t]; io.out[t] = out[t]; io.dim[t] = dims[t];
    }
    SMK_REQUIRE(dims[4] == 3, "smk_cycle_augment: jaw_params must have 3 columns");
    SMK_REQUIRE(dims[3] >= h->n_exp, "smk_cycle_augment: expression width %d < the templates' %d columns", dims[3], h->n_exp);
    const SmkCycleDraws d = dbg ? *dbg : SmkCycleDraws{};
    cudaStream_t st = (cudaStream_t)stream;
    const int R = B * Ke;
    SMK_TAG("cycle_augment", 4.0 * R * (dims[0] + dims[1] + dims[2] + 2 * (dims[3] + 5)), 0.0, st);
    SMK_LAUNCH(cycle_augment_kernel, dim3(1), dim3(kThreads), 0, st, io, B, R, use_eyelids, (const float*)h->rows, (const int*)h->offsets,
               h->n_keys, h->n_exp, rng_state, d);
    SMK_CHECK_LAUNCH();
    return 0;
}
