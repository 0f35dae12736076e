// Masking step between Renderer and SmirkGenerator (SURVEY.md §8f #1) — reference src/utils/masking.py and its call
// site demo.py:138-167.  WORK IN PROGRESS: written against oracle/masking_ref.py and tests/golden/masking.npz, not yet
// run on a GPU (branch wip/masking-kernels).
//
// Randomness stays where the reference has it — in torch (multinomial / rand / randn / bernoulli on the caller's
// generator); everything that is deterministic given those draws runs here:
//   smk_masking_face_weights   masking.py:146-160  per-face sampling weight = (mean z of the 3 vertex normals < 0.05 ?
//                                                  base weight : 0) x projected area; vertex normals accumulated in
//                                                  the reference's index_add_ order (util.py:30-62)
//   smk_masking_points         masking.py:166-174  barycentric points of the sampled faces -> clamped integer pixels
//   smk_masking_compose        demo.py:154-160 + masking.py:71-102: point mask, 21x21 dilation of the hull mask
//                              (1 - maxpool(1 - mask)), x (1 - rendered_mask), noise on the retained points, 11x11
//                              patches knocked out around random centres, composite — three launches, two of them the
//                              separable halves of the max-pools.
// (2) smk_masking_forward chains them into the whole demo.py:138-165 step with the draws made ON the device by a
// counter-based generator (Philox4x32-10 keyed by (seed, counter, element)): multinomial face sampling by inverse CDF,
// uniform barycentrics, the per-image point budget `rbound`, the Gaussian pixel noise and the Bernoulli patch centres.
// The reference draws from torch's global RNG, so only distributional parity with it is possible (SURVEY.md §8f #1);
// what IS exact: given the draws this call exports (optional debug outputs), the masked image equals the reference's
// `masking()` fed the same draws.  The counter lives in device memory and is advanced by the last kernel, so a captured
// CUDA graph produces fresh draws on every replay.
// (3) smk_masking_train_forward (include/smirk_b200.h) runs the trainer's step1 / step2 masking on the same kernels:
// every sampled point kept (no rbound), transfer_pixels between two meshes, Ke repeats read as row r mod B (`Bsrc`).
// All of it is HBM-bound byte/float shuffling over [B,3,224,224] images (602 KB per face in, 602 KB out).
#include "common.cuh"
#include "philox.cuh"
#include <math.h>
#include <algorithm>
#include <vector>

namespace {

using smk::U4;
using smk::philox;
using smk::u01;

struct MaskDev {
    int V, F;
    int32_t* faces;        // [F][3]
    int32_t* adj_ptr;      // [V+1]  CSR vertex -> (face<<2 | corner) in the order of the reference's three index_add_ passes
    int32_t* adj;
};

// vertex normals of the full mesh (util.vertex_normals), one thread per vertex, fixed accumulation order
__global__ void __launch_bounds__(128)
mask_normals_kernel(MaskDev d, const float* __restrict__ tv, int B, float* __restrict__ normals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= d.V) return;
    const float* vb = tv + (size_t)b * d.V * 3;
    float nx = 0.f, ny = 0.f, nz = 0.f;
    for (int e = d.adj_ptr[i]; e < d.adj_ptr[i + 1]; ++e) {
        const int code = d.adj[e], f = code >> 2, c = code & 3;
        const int32_t* tri = d.faces + (size_t)f * 3;
        const float* p = vb + (size_t)tri[c] * 3;
        const float* q1 = vb + (size_t)tri[(c + 1) % 3] * 3;
        const float* q2 = vb + (size_t)tri[(c + 2) % 3] * 3;
        const float ax = __fsub_rn(q1[0], p[0]), ay = __fsub_rn(q1[1], p[1]), az = __fsub_rn(q1[2], p[2]);
        const float bx = __fsub_rn(q2[0], p[0]), by = __fsub_rn(q2[1], p[1]), bz = __fsub_rn(q2[2], p[2]);
        nx = __fadd_rn(nx, __fsub_rn(__fmul_rn(ay, bz), __fmul_rn(az, by)));
        ny = __fadd_rn(ny, __fsub_rn(__fmul_rn(az, bx), __fmul_rn(ax, bz)));
        nz = __fadd_rn(nz, __fsub_rn(__fmul_rn(ax, by), __fmul_rn(ay, bx)));
    }
    const float len = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
    const float den = fmaxf(len, 1e-6f);
    float* n = normals + ((size_t)b * d.V + i) * 3;
    n[0] = __fdiv_rn(nx, den); n[1] = __fdiv_rn(ny, den); n[2] = __fdiv_rn(nz, den);
}

__global__ void __launch_bounds__(128)
mask_face_weights_kernel(MaskDev d, const float* __restrict__ tv, const float* __restrict__ normals,
                         const float* __restrict__ base_prob, int B, float* __restrict__ w) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (f >= d.F) return;
    const int32_t* tri = d.faces + (size_t)f * 3;
    const float* nb = normals + (size_t)b * d.V * 3;
    const float* vb = tv + (size_t)b * d.V * 3;
    // mean over the three corners (torch: sum / 3)
    const float fnz = __fdiv_rn(__fadd_rn(__fadd_rn(nb[(size_t)tri[0] * 3 + 2], nb[(size_t)tri[1] * 3 + 2]), nb[(size_t)tri[2] * 3 + 2]), 3.0f);
    const float x1 = vb[(size_t)tri[0] * 3], y1 = vb[(size_t)tri[0] * 3 + 1];
    const float x2 = vb[(size_t)tri[1] * 3], y2 = vb[(size_t)tri[1] * 3 + 1];
    const float x3 = vb[(size_t)tri[2] * 3], y3 = vb[(size_t)tri[2] * 3 + 1];
    // 0.5 * |x1 y2 + x2 y3 + x3 y1 - x2 y1 - x3 y2 - x1 y3|, left to right (masking.py:50)
    float s = __fadd_rn(__fadd_rn(__fmul_rn(x1, y2), __fmul_rn(x2, y3)), __fmul_rn(x3, y1));
    s = __fsub_rn(__fsub_rn(__fsub_rn(s, __fmul_rn(x2, y1)), __fmul_rn(x3, y2)), __fmul_rn(x1, y3));
    const float area = __fmul_rn(0.5f, fabsf(s));
    const float p = fnz < 0.05f ? base_prob[f] : 0.0f;
    w[(size_t)b * d.F + f] = __fmul_rn(p, area);
}

__global__ void __launch_bounds__(256)
mask_points_kernel(MaskDev d, const float* __restrict__ tv, const int64_t* __restrict__ fidx, const float* __restrict__ bary,
                   int B, int Bsrc, int N, int S, int64_t* __restrict__ npoints) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * N) return;
    const int b = (int)(i / N);
    const long src = (long)(b % Bsrc) * N + (i - (long)b * N);                          // draws of row b mod Bsrc
    const int32_t* tri = d.faces + (size_t)fidx[src] * 3;
    const float* vb = tv + (size_t)b * d.V * 3;
    const float b0 = bary[src * 3], b1 = bary[src * 3 + 1], b2 = bary[src * 3 + 2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        float p = __fmul_rn(vb[(size_t)tri[0] * 3 + k], b0);
        p = fmaf(vb[(size_t)tri[1] * 3 + k], b1, p);
        p = fmaf(vb[(size_t)tri[2] * 3 + k], b2, p);
        const float v = __fmul_rn(__fmul_rn(0.5f, __fadd_rn(1.0f, p)), (float)S);         // .5 * (1 + p) * S
        long q = (long)v;                                                                 // .long(): truncation
        q = q < 0 ? 0 : (q > S - 1 ? S - 1 : q);
        npoints[i * 2 + k] = q;
    }
}

__global__ void __launch_bounds__(256)
mask_scatter_kernel(const int64_t* __restrict__ npoints, const int64_t* __restrict__ rbound, int B, int N, int S, uint8_t* __restrict__ pm) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * N) return;
    const int b = (int)(i / N), j = (int)(i - (long)b * N);
    if (j >= rbound[b]) return;
    pm[((size_t)b * S + npoints[i * 2 + 1]) * S + npoints[i * 2]] = 1;                    // all writers store the same value
}

// horizontal halves of the two max-pools: th = max_{|dx|<=wr}(1 - hull), tc = max_{|dx|<=5} centres (OOB ignored, like
// max_pool2d's -inf padding)
__global__ void __launch_bounds__(256)
mask_hmax_kernel(const float* __restrict__ hull, const float* __restrict__ centres, int B, int Bsrc, int S, int wr,
                 float* __restrict__ th, float* __restrict__ tc) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * S * S) return;
    const int x = (int)(i % S);
    const long plane = (long)S * S, b = i / plane;
    const float* hr = hull + (b % Bsrc) * plane + (i - b * plane - x);                  // hull of image b mod Bsrc
    float m = -INFINITY;
    for (int dx = -wr; dx <= wr; ++dx) { const int xx = x + dx; if (xx >= 0 && xx < S) m = fmaxf(m, __fsub_rn(1.0f, hr[xx])); }
    th[i] = m;
    if (centres) {
        const float* cr = centres + (i - x);
        float c = -INFINITY;
        for (int dx = -5; dx <= 5; ++dx) { const int xx = x + dx; if (xx >= 0 && xx < S) c = fmaxf(c, cr[xx]); }
        tc[i] = c;
    }
}

// vertical halves + composite (masking.py:79-100)
__global__ void __launch_bounds__(256)
mask_compose_kernel(const float* __restrict__ img, const float* __restrict__ th, const float* __restrict__ tc,
                    const uint8_t* __restrict__ pm, const float* __restrict__ extra, const float* __restrict__ rendered_mask,
                    const float* __restrict__ noise_mult, int B, int Bsrc, int S, int wr, float* __restrict__ out) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * S * S) return;
    const int b = (int)(i / ((long)S * S));
    const int pix = (int)(i - (long)b * S * S), y = pix / S, x = pix - y * S;
    const float* tcol = th + (size_t)b * S * S + x;
    float m = -INFINITY;
    for (int dy = -wr; dy <= wr; ++dy) { const int yy = y + dy; if (yy >= 0 && yy < S) m = fmaxf(m, tcol[(size_t)yy * S]); }
    float mask = __fsub_rn(1.0f, m);
    if (rendered_mask) mask = __fmul_rn(mask, __fsub_rn(1.0f, rendered_mask[i]));
    float keep = 1.0f;
    if (tc) {
        const float* ccol = tc + (size_t)b * S * S + x;
        float c = -INFINITY;
        for (int dy = -5; dy <= 5; ++dy) { const int yy = y + dy; if (yy >= 0 && yy < S) c = fmaxf(c, ccol[(size_t)yy * S]); }
        keep = __fsub_rn(1.0f, c);
    }
    const float on = (pm && pm[i]) ? 1.0f : 0.0f;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const size_t o = ((size_t)b * 3 + ch) * S * S + pix;
        const float v = img[((size_t)(b % Bsrc) * 3 + ch) * S * S + pix];              // image b mod Bsrc
        float e = extra ? extra[o] : __fmul_rn(v, on);                // extra_points: given (masking.py:71), or img * pmask (demo.py:162)
        if (noise_mult) e = __fmul_rn(e, noise_mult[o]);
        if (tc) e = __fmul_rn(e, keep);
        out[o] = e > 0.0f ? e : __fmul_rn(v, mask);
    }
}


// one CTA per image: inclusive CDF of the face weights in shared memory, N inverse-CDF samples, barycentrics, rbound
__global__ void __launch_bounds__(512)
mask_sample_kernel(const float* __restrict__ w, int F, int N, float ratio_mul, const uint64_t* __restrict__ rng,
                   int64_t* __restrict__ fidx, float* __restrict__ bary, int64_t* __restrict__ rbound) {
    extern __shared__ float cdf[];                      // [F]
    __shared__ float part[512];
    const int b = blockIdx.x, t = threadIdx.x, nt = blockDim.x;
    const float* wb = w + (size_t)b * F;
    const int per = (F + nt - 1) / nt, lo = t * per, hi = min(F, lo + per);
    float s = 0.f;
    for (int i = lo; i < hi; ++i) { s += fmaxf(wb[i], 0.f); cdf[i] = s; }
    part[t] = s;
    __syncthreads();
    for (int off = 1; off < nt; off <<= 1) {            // Hillis-Steele scan of the per-thread totals
        float v = t >= off ? part[t - off] : 0.f;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    const float base = t > 0 ? part[t - 1] : 0.f;
    for (int i = lo; i < hi; ++i) cdf[i] += base;
    __syncthreads();
    const float total = part[nt - 1];
    const uint64_t seed = rng[0], ctr = rng[1];
    for (int j = t; j < N; j += nt) {
        const U4 r = philox(seed, ctr, 0u, (uint32_t)b, (uint32_t)j);
        int f = 0;
        if (total > 0.f) {
            const float x = u01(r.x) * total;
            int a = 0, c = F - 1;                       // first index with cdf > x
            while (a < c) { const int m = (a + c) >> 1; if (cdf[m] > x) c = m; else a = m + 1; }
            f = a;
            // the segmented float scan may be non-monotone by an ulp at a segment seam: never hand out a zero-weight face
            while (f < F - 1 && !(wb[f] > 0.f)) ++f;
            while (f > 0 && !(wb[f] > 0.f)) --f;
        }
        float u = u01(r.y), v = u01(r.z);
        if (u + v > 1.f) { u = 1.f - u; v = 1.f - v; }  // masking.py:61-66: reflect into the triangle
        const size_t o = (size_t)b * N + j;
        fidx[o] = f;
        bary[o * 3] = 1.f - (u + v); bary[o * 3 + 1] = u; bary[o * 3 + 2] = v;
    }
    if (t == 0 && rbound) {                             // demo.py:151-153
        const U4 r = philox(seed, ctr, 1u, (uint32_t)b, 0u);
        const float rsign = (r.x & 1u) ? 1.f : -1.f;
        const float rscale = u01(r.y) * (ratio_mul - 1.f) + 1.f;
        rbound[b] = (int64_t)((float)N * (1.f / ratio_mul) * powf(rscale, rsign));
    }
}

// noise_mult[b,c,y,x] = N(0,1) * 0.05 + 1 (masking.py:84-86); centres[b,0,y,x] ~ Bernoulli(p) (masking.py:89-92)
__global__ void __launch_bounds__(256)
mask_rng_fill_kernel(int B, int S, float p_centre, const uint64_t* __restrict__ rng, float* __restrict__ noise, float* __restrict__ centres) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long npx = (long)B * S * S;
    if (i >= npx) return;
    const uint64_t seed = rng[0], ctr = rng[1];
    const U4 r = philox(seed, ctr, 2u, (uint32_t)(i >> 32), (uint32_t)i);
    const U4 q = philox(seed, ctr, 3u, (uint32_t)(i >> 32), (uint32_t)i);
    const int b = (int)(i / ((long)S * S)); const long pix = i - (long)b * S * S;
    // Box-Muller: two uniforms -> two normals; three channels use (r.x,r.y) cos / sin and (r.z,r.w) cos
    const float m0 = sqrtf(-2.f * logf(1.f - u01(r.x))), a0 = 6.2831853f * u01(r.y);
    const float m1 = sqrtf(-2.f * logf(1.f - u01(r.z))), a1 = 6.2831853f * u01(r.w);
    const float n[3] = {m0 * cosf(a0), m0 * sinf(a0), m1 * cosf(a1)};
#pragma unroll
    for (int c = 0; c < 3; ++c) noise[((size_t)b * 3 + c) * S * S + pix] = fmaf(n[c], 0.05f, 1.0f);
    centres[i] = u01(q.x) < p_centre ? 1.f : 0.f;
}

// all_positive = 0: rendered_mask = 1 - all(rendered == 0 over channels)   (demo.py:146, smirk_trainer.py:77)
// all_positive = 1: rendered_mask = all(rendered > 0 over channels)          (smirk_trainer.py:290)
// Neither is the complement of the other: a pixel with one zero channel is 1 under the first rule and 0 under the second.
__global__ void __launch_bounds__(256)
mask_rendered_kernel(const float* __restrict__ rendered, int B, int S, int all_positive, float* __restrict__ rmask) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * S * S) return;
    const int b = (int)(i / ((long)S * S)); const long pix = i - (long)b * S * S;
    const float* r = rendered + (size_t)b * 3 * S * S + pix;
    const float r0 = r[0], r1 = r[(size_t)S * S], r2 = r[(size_t)2 * S * S];
    if (all_positive) { rmask[i] = (r0 > 0.f && r1 > 0.f && r2 > 0.f) ? 1.f : 0.f; return; }
    const bool bg = r0 == 0.f && r1 == 0.f && r2 == 0.f;
    rmask[i] = bg ? 0.f : 1.f;
}

__global__ void mask_rng_advance_kernel(uint64_t* rng) { if (threadIdx.x == 0) rng[1] += 1; }

// transfer_pixels (masking.py:116-129): out[b, :, p2.y, p2.x] = img[b, :, p1.y, p1.x] for the first rbound[b] (or all) point
// pairs; with duplicate targets the LAST pair in index order wins (the sequential semantics of the reference's indexed
// assignment).  Pass 1: winner[target pixel] = max pair index (atomicMax); pass 2: every pixel copies from its winner.
__global__ void __launch_bounds__(256)
mask_transfer_winner_kernel(const int64_t* __restrict__ p2, const int64_t* __restrict__ rbound, int B, int N, int S, int* __restrict__ winner) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * N) return;
    const int b = (int)(i / N), j = (int)(i - (long)b * N);
    if (rbound && j >= rbound[b]) return;
    const int64_t x = p2[i * 2], y = p2[i * 2 + 1];
    if (x < 0 || x >= S || y < 0 || y >= S) return;
    atomicMax(winner + ((size_t)b * S + y) * S + x, j);
}
__global__ void __launch_bounds__(256)
mask_transfer_copy_kernel(const float* __restrict__ img, const int64_t* __restrict__ p1, const int* __restrict__ winner, int B, int Bsrc, int N, int S,
                          float* __restrict__ out) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * S * S) return;
    const int b = (int)(i / ((long)S * S)); const long pix = i - (long)b * S * S;
    const int bs = b % Bsrc;                            // source image and points1 of row b: row b mod Bsrc
    const int j = winner[i];
    int64_t sx = 0, sy = 0;
    if (j >= 0) { sx = p1[((size_t)bs * N + j) * 2]; sy = p1[((size_t)bs * N + j) * 2 + 1]; }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        out[((size_t)b * 3 + ch) * S * S + pix] = j >= 0 ? img[((size_t)bs * 3 + ch) * S * S + (size_t)sy * S + sx] : 0.f;
    }
}

}  // namespace

struct SmkMasking {
    MaskDev d;
    smk::DeviceArena arena;
};

extern "C" int smk_masking_create(const SmkMaskingDesc* desc, SmkMasking** out) {
    SMK_REQUIRE(desc && out && desc->faces, "smk_masking_create: null argument");
    SMK_REQUIRE(desc->n_verts > 0 && desc->n_faces > 0, "smk_masking_create: empty mesh");
    SmkMasking* h = new SmkMasking();
    MaskDev& d = h->d;
    d.V = desc->n_verts; d.F = desc->n_faces;
    for (int i = 0; i < d.F * 3; ++i)
        if (desc->faces[i] < 0 || desc->faces[i] >= d.V) { delete h; smk::set_error("smk_masking_create: face index out of range"); return -1; }
    std::vector<int32_t> ptr(d.V + 1, 0), adj((size_t)d.F * 3);
    for (int i = 0; i < d.F * 3; ++i) ptr[desc->faces[i] + 1]++;
    for (int i = 0; i < d.V; ++i) ptr[i + 1] += ptr[i];
    std::vector<int32_t> fill(ptr.begin(), ptr.end() - 1);
    const int order[3] = {1, 2, 0};                                    // util.py:52-57: corner 1, then 2, then 0; faces ascending
    for (int pass = 0; pass < 3; ++pass)
        for (int f = 0; f < d.F; ++f) { const int c = order[pass]; adj[fill[desc->faces[f * 3 + c]]++] = (f << 2) | c; }
    cudaError_t e = h->arena.upload(desc->faces, (size_t)d.F * 3, &d.faces);
    if (e == cudaSuccess) e = h->arena.upload(ptr, &d.adj_ptr);
    if (e == cudaSuccess) e = h->arena.upload(adj, &d.adj);
    if (e != cudaSuccess) { smk::set_error("smk_masking_create: upload failed: %s", cudaGetErrorString(e)); delete h; return (int)e; }
    *out = h;
    return 0;
}

extern "C" void smk_masking_destroy(SmkMasking* h) { delete h; }

extern "C" size_t smk_masking_workspace_bytes(const SmkMasking* h, int B, int S) {
    const size_t b = (size_t)(B > 0 ? B : 1);
    return smk::ws_round(b * h->d.V * 3 * sizeof(float)) + 2 * smk::ws_round(b * S * S * sizeof(float)) + smk::ws_round(b * S * S);
}

extern "C" int smk_masking_face_weights(const SmkMasking* h, const float* trans_verts, const float* base_prob, int B,
                                        float* weights, void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;
    SMK_REQUIRE(h && trans_verts && base_prob && weights, "smk_masking_face_weights: null argument");
    SMK_REQUIRE(ws && ws_bytes >= smk::ws_round((size_t)B * h->d.V * 3 * sizeof(float)), "smk_masking_face_weights: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    float* normals = reinterpret_cast<float*>(ws);
    const MaskDev& d = h->d;
    SMK_TAG("mask_normals", 24.0 * B * d.V + 12.0 * d.F, 0.0, st);
    SMK_LAUNCH(mask_normals_kernel, dim3(smk::cdiv(d.V, 128), B), dim3(128), 0, st, d, trans_verts, B, normals);
    SMK_CHECK_LAUNCH();
    SMK_TAG("mask_face_weights", 4.0 * B * d.F + 24.0 * B * d.V, 0.0, st);
    SMK_LAUNCH(mask_face_weights_kernel, dim3(smk::cdiv(d.F, 128), B), dim3(128), 0, st, d, trans_verts, (const float*)normals, base_prob, B, weights);
    SMK_CHECK_LAUNCH();
    return 0;
}

namespace {

int points_impl(const SmkMasking* h, const float* tv, const int64_t* fidx, const float* bary, int B, int Bsrc, int N, int S,
                int64_t* npoints, cudaStream_t st) {
    SMK_TAG("mask_points", 36.0 * B * N, 0.0, st);
    SMK_LAUNCH(mask_points_kernel, dim3(smk::cdiv((long)B * N, 256)), dim3(256), 0, st, h->d, tv, fidx, bary, B, Bsrc, N, S, npoints);
    SMK_CHECK_LAUNCH();
    return 0;
}

// winner: B*S*S ints of scratch
int transfer_impl(const float* img, const int64_t* points1, const int64_t* points2, const int64_t* rbound, int B, int Bsrc, int N, int S,
                  float* out, int* winner, cudaStream_t st) {
    SMK_CHECK_CUDA(cudaMemsetAsync(winner, 0xFF, (size_t)B * S * S * sizeof(int), st));        // -1
    if (N > 0) {
        SMK_TAG("mask_transfer_winner", 20.0 * B * N, 0.0, st);
        SMK_LAUNCH(mask_transfer_winner_kernel, dim3(smk::cdiv((long)B * N, 256)), dim3(256), 0, st, points2, rbound, B, N, S, winner);
        SMK_CHECK_LAUNCH();
    }
    SMK_TAG("mask_transfer_copy", 4.0 * B * S * S * 5.0, 0.0, st);
    SMK_LAUNCH(mask_transfer_copy_kernel, dim3(smk::cdiv((long)B * S * S, 256)), dim3(256), 0, st, img, points1, (const int*)winner, B, Bsrc, N, S, out);
    SMK_CHECK_LAUNCH();
    return 0;
}

// ws: smk_masking_workspace_bytes(h, B, S); img and hull rows are those of image b mod Bsrc
int compose_impl(const SmkMasking* h, const float* img, const float* hull, const int64_t* npoints, const int64_t* rbound, int N,
                 const float* extra_points, const float* rendered_mask, const float* noise_mult, const float* random_centres,
                 int wr, int B, int Bsrc, int S, float* masked, void* ws, size_t ws_bytes, cudaStream_t st) {
    if (extra_points) N = 0;                            // the caller supplies extra_points (masking.py:71); no point mask to build
    smk::Workspace w(ws, ws_bytes);
    w.take<float>((size_t)B * h->d.V * 3);                              // (normals slot, unused here)
    float* th = w.take<float>((size_t)B * S * S);
    float* tc = w.take<float>((size_t)B * S * S);
    uint8_t* pm = w.take<uint8_t>((size_t)B * S * S);
    SMK_REQUIRE(pm != nullptr, "smk_masking_compose: workspace carve-up failed");
    SMK_CHECK_CUDA(cudaMemsetAsync(pm, 0, (size_t)B * S * S, st));
    const long npx = (long)B * S * S;
    if (N > 0) {
        SMK_TAG("mask_scatter", 24.0 * B * N, 0.0, st);
        SMK_LAUNCH(mask_scatter_kernel, dim3(smk::cdiv((long)B * N, 256)), dim3(256), 0, st, npoints, rbound, B, N, S, pm);
        SMK_CHECK_LAUNCH();
    }
    SMK_TAG("mask_hmax", 16.0 * npx, 0.0, st);
    SMK_LAUNCH(mask_hmax_kernel, dim3(smk::cdiv(npx, 256)), dim3(256), 0, st, hull, random_centres, B, Bsrc, S, wr, th, tc);
    SMK_CHECK_LAUNCH();
    SMK_TAG("mask_compose", 4.0 * npx * (3 + 3 + 2 + (noise_mult ? 3 : 0)), 0.0, st);
    SMK_LAUNCH(mask_compose_kernel, dim3(smk::cdiv(npx, 256)), dim3(256), 0, st, img, (const float*)th, (const float*)(random_centres ? tc : nullptr),
               (const uint8_t*)pm, extra_points, rendered_mask, noise_mult, B, Bsrc, S, wr, masked);
    SMK_CHECK_LAUNCH();
    return 0;
}

// The face weights of trans_verts [B] and N inverse-CDF samples per image into fidx / bary; rbound NULL = keep every point.
int sample_impl(const SmkMasking* h, const float* tv, const float* base_prob, int B, int N, float ratio_mul, const uint64_t* rng,
                float* weights, int64_t* fidx, float* bary, int64_t* rbound, void* ws, size_t ws_bytes, cudaStream_t st) {
    const MaskDev& d = h->d;
    if (int rc = smk_masking_face_weights(h, tv, base_prob, B, weights, ws, ws_bytes, st)) return rc;
    SMK_CHECK_CUDA(smk::set_max_dynamic_smem<mask_sample_kernel>(160 * 1024));
    SMK_TAG("mask_sample", 4.0 * B * d.F + 36.0 * B * N, 0.0, st);
    SMK_LAUNCH(mask_sample_kernel, dim3(B), dim3(512), (size_t)d.F * sizeof(float), st, (const float*)weights, d.F, N, ratio_mul,
               rng, fidx, bary, rbound);
    SMK_CHECK_LAUNCH();
    return 0;
}

}  // namespace

extern "C" int smk_masking_points(const SmkMasking* h, const float* trans_verts, const int64_t* face_idx, const float* bary,
                                  int B, int N, int image_size, int64_t* npoints, void* stream) {
    if (B == 0 || N == 0) return 0;
    SMK_REQUIRE(h && trans_verts && face_idx && bary && npoints && image_size > 0, "smk_masking_points: bad argument");
    return points_impl(h, trans_verts, face_idx, bary, B, B, N, image_size, npoints, (cudaStream_t)stream);
}

extern "C" int smk_masking_transfer_pixels(const float* img, const int64_t* points1, const int64_t* points2, const int64_t* rbound,
                                           int B, int N, int S, float* out, void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;
    SMK_REQUIRE(img && out && (N == 0 || (points1 && points2)) && S > 0, "smk_masking_transfer_pixels: bad argument");
    SMK_REQUIRE(ws && ws_bytes >= (size_t)B * S * S * sizeof(int), "smk_masking_transfer_pixels: workspace too small (B*S*S ints)");
    return transfer_impl(img, points1, points2, rbound, B, B, N, S, out, reinterpret_cast<int*>(ws), (cudaStream_t)stream);
}

extern "C" int smk_masking_compose(const SmkMasking* h, const float* img, const float* hull, const int64_t* npoints, const int64_t* rbound,
                                   int N, const float* extra_points, const float* rendered_mask, const float* noise_mult, const float* random_centres,
                                   int wr, int B, int S, float* masked, void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;
    SMK_REQUIRE(h && img && hull && masked && (N == 0 || extra_points || (npoints && rbound)) && wr >= 0 && S > 0, "smk_masking_compose: bad argument");
    SMK_REQUIRE(ws && ws_bytes >= smk_masking_workspace_bytes(h, B, S), "smk_masking_compose: workspace too small");
    return compose_impl(h, img, hull, npoints, rbound, N, extra_points, rendered_mask, noise_mult, random_centres, wr, B, B, S, masked, ws,
                        ws_bytes, (cudaStream_t)stream);
}

extern "C" size_t smk_masking_forward_workspace_bytes(const SmkMasking* h, int B, int S, int N) {
    const size_t b = (size_t)(B > 0 ? B : 1), px = b * S * S;
    return smk_masking_workspace_bytes(h, B, S) + smk::ws_round(b * h->d.F * sizeof(float)) + smk::ws_round(b * N * 8) + smk::ws_round(b * N * 12) +
           smk::ws_round(b * N * 16) + smk::ws_round(b * 8) + smk::ws_round(px * 12) + 2 * smk::ws_round(px * 4) + 4096;
}

extern "C" int smk_masking_forward(const SmkMasking* h, const float* img, const float* hull, const float* trans_verts, const float* rendered,
                                   const float* base_prob, int B, int S, int N, int wr, float ratio_mul, float p_centre, int extra_noise,
                                   uint64_t* rng_state, float* masked, int64_t* dbg_face_idx, float* dbg_bary, int64_t* dbg_npoints,
                                   int64_t* dbg_rbound, float* dbg_noise, float* dbg_centres, void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;
    SMK_REQUIRE(h && img && hull && trans_verts && rendered && base_prob && rng_state && masked, "smk_masking_forward: null argument");
    SMK_REQUIRE(N > 0 && S > 0 && wr >= 0 && ratio_mul >= 1.f, "smk_masking_forward: bad sizes");
    SMK_REQUIRE(ws && ws_bytes >= smk_masking_forward_workspace_bytes(h, B, S, N), "smk_masking_forward: workspace too small");
    SMK_REQUIRE((size_t)h->d.F * sizeof(float) <= 160 * 1024, "smk_masking_forward: too many faces for the shared-memory CDF");
    cudaStream_t st = (cudaStream_t)stream;
    const MaskDev& d = h->d;
    const size_t base = smk_masking_workspace_bytes(h, B, S);
    smk::Workspace w((char*)ws + base, ws_bytes - base);
    const long npx = (long)B * S * S;
    float* weights = w.take<float>((size_t)B * d.F);
    int64_t* fidx = dbg_face_idx ? dbg_face_idx : w.take<int64_t>((size_t)B * N);
    float* bary = dbg_bary ? dbg_bary : w.take<float>((size_t)B * N * 3);
    int64_t* npoints = dbg_npoints ? dbg_npoints : w.take<int64_t>((size_t)B * N * 2);
    int64_t* rbound = dbg_rbound ? dbg_rbound : w.take<int64_t>((size_t)B);
    float* noise = dbg_noise ? dbg_noise : w.take<float>((size_t)npx * 3);
    float* centres = dbg_centres ? dbg_centres : w.take<float>((size_t)npx);
    float* rmask = w.take<float>((size_t)npx);
    SMK_REQUIRE(rmask != nullptr, "smk_masking_forward: workspace carve-up failed");
    if (int rc = sample_impl(h, trans_verts, base_prob, B, N, ratio_mul, rng_state, weights, fidx, bary, rbound, ws, base, st)) return rc;
    if (int rc = points_impl(h, trans_verts, fidx, bary, B, B, N, S, npoints, st)) return rc;
    SMK_TAG("mask_rng_fill", 16.0 * npx, 0.0, st);
    SMK_LAUNCH(mask_rng_fill_kernel, dim3(smk::cdiv(npx, 256)), dim3(256), 0, st, B, S, p_centre, (const uint64_t*)rng_state, noise, centres);
    SMK_CHECK_LAUNCH();
    SMK_TAG("mask_rendered", 16.0 * npx, 0.0, st);
    SMK_LAUNCH(mask_rendered_kernel, dim3(smk::cdiv(npx, 256)), dim3(256), 0, st, rendered, B, S, 0, rmask);
    SMK_CHECK_LAUNCH();
    if (int rc = compose_impl(h, img, hull, npoints, rbound, N, nullptr, rmask, extra_noise ? noise : nullptr, p_centre > 0.f ? centres : nullptr,
                              wr, B, B, S, masked, ws, base, st)) return rc;
    SMK_TAG("mask_rng_advance", 16.0, 0.0, st);
    SMK_LAUNCH(mask_rng_advance_kernel, dim3(1), dim3(32), 0, st, rng_state);
    SMK_CHECK_LAUNCH();
    return 0;
}

// ---- the trainer's masking (include/smirk_b200.h) ----
extern "C" size_t smk_masking_train_workspace_bytes(const SmkMasking* h, int B, int Ke, int S, int N) {
    if (!h) return 0;
    const size_t b = (size_t)(B > 0 ? B : 1), r = b * (size_t)(Ke > 0 ? Ke : 1), px = r * S * S, n = (size_t)(N > 0 ? N : 1);
    return smk_masking_workspace_bytes(h, (int)r, S) + smk::ws_round(b * h->d.F * sizeof(float)) + smk::ws_round(b * n * 8) +
           smk::ws_round(b * n * 12) + smk::ws_round(b * n * 16) + smk::ws_round(r * n * 16) + smk::ws_round(px * 12) +
           smk::ws_round(px * 12) + 3 * smk::ws_round(px * 4) + 4096;
}

extern "C" int smk_masking_train_forward(const SmkMasking* h, int step, const float* img, const float* hull, const float* tv_first,
                                         const float* tv_second, const float* rendered, const float* base_prob, int B, int Ke, int S, int N,
                                         int wr, float p_centre, uint64_t* rng_state, float* masked, int64_t* dbg_face_idx, float* dbg_bary,
                                         int64_t* dbg_points1, int64_t* dbg_points2, float* dbg_noise, float* dbg_centres, void* ws,
                                         size_t ws_bytes, void* stream) {
    SMK_REQUIRE(step == 1 || step == 2, "smk_masking_train_forward: step must be 1 or 2");
    SMK_REQUIRE(B >= 0 && Ke >= 1 && (step == 2 || Ke == 1), "smk_masking_train_forward: bad batch (B >= 0, Ke >= 1, step 1 needs Ke == 1)");
    if (B == 0) return 0;
    SMK_REQUIRE(h && img && hull && tv_first && rendered && base_prob && rng_state && masked, "smk_masking_train_forward: null argument");
    SMK_REQUIRE((step == 2) == (tv_second != nullptr), "smk_masking_train_forward: tv_second is required by step 2 and only by it");
    SMK_REQUIRE(N > 0 && S > 0 && wr >= 0 && p_centre >= 0.f && p_centre <= 1.f, "smk_masking_train_forward: bad sizes");
    SMK_REQUIRE(ws && ws_bytes >= smk_masking_train_workspace_bytes(h, B, Ke, S, N), "smk_masking_train_forward: workspace too small");
    SMK_REQUIRE((size_t)h->d.F * sizeof(float) <= 160 * 1024, "smk_masking_train_forward: too many faces for the shared-memory CDF");
    cudaStream_t st = (cudaStream_t)stream;
    const MaskDev& d = h->d;
    const int R = B * Ke;
    const long npx = (long)R * S * S;
    const size_t base = smk_masking_workspace_bytes(h, R, S);
    smk::Workspace w((char*)ws + base, ws_bytes - base);
    float* weights = w.take<float>((size_t)B * d.F);
    int64_t* fidx = dbg_face_idx ? dbg_face_idx : w.take<int64_t>((size_t)B * N);
    float* bary = dbg_bary ? dbg_bary : w.take<float>((size_t)B * N * 3);
    int64_t* points1 = dbg_points1 ? dbg_points1 : w.take<int64_t>((size_t)B * N * 2);
    int64_t* points2 = step == 1 ? points1 : (dbg_points2 ? dbg_points2 : w.take<int64_t>((size_t)R * N * 2));
    float* extra = w.take<float>((size_t)npx * 3);
    float* noise = dbg_noise ? dbg_noise : w.take<float>((size_t)npx * 3);
    float* centres = dbg_centres ? dbg_centres : w.take<float>((size_t)npx);
    float* rmask = w.take<float>((size_t)npx);
    int* winner = w.take<int>((size_t)npx);
    SMK_REQUIRE(winner != nullptr && points2 != nullptr, "smk_masking_train_forward: workspace carve-up failed");
    // smirk_trainer.py:80-84 / 268-271: all int(mask_ratio * S^2) samples are kept (no rbound)
    if (int rc = sample_impl(h, tv_first, base_prob, B, N, 1.f, rng_state, weights, fidx, bary, nullptr, ws, base, st)) return rc;
    if (int rc = points_impl(h, tv_first, fidx, bary, B, B, N, S, points1, st)) return rc;
    if (step == 2)                                      // :275-283: the same draws (repeated Ke times) on the second path's mesh
        if (int rc = points_impl(h, tv_second, fidx, bary, R, B, N, S, points2, st)) return rc;
    // :87 transfer_pixels(img, npoints, npoints) / :287 transfer_pixels(img.repeat(Ke), points1.repeat(Ke), points2)
    if (int rc = transfer_impl(img, points1, points2, nullptr, R, B, N, S, extra, winner, st)) return rc;
    SMK_TAG("mask_rng_fill", 16.0 * npx, 0.0, st);
    SMK_LAUNCH(mask_rng_fill_kernel, dim3(smk::cdiv(npx, 256)), dim3(256), 0, st, R, S, p_centre, (const uint64_t*)rng_state, noise, centres);
    SMK_CHECK_LAUNCH();
    SMK_TAG("mask_rendered", 16.0 * npx, 0.0, st);
    SMK_LAUNCH(mask_rendered_kernel, dim3(smk::cdiv(npx, 256)), dim3(256), 0, st, rendered, R, S, step == 2 ? 1 : 0, rmask);
    SMK_CHECK_LAUNCH();
    if (int rc = compose_impl(h, img, hull, nullptr, nullptr, 0, extra, rmask, noise, p_centre > 0.f ? centres : nullptr, wr, R, B, S,
                              masked, ws, base, st)) return rc;
    SMK_TAG("mask_rng_advance", 16.0, 0.0, st);
    SMK_LAUNCH(mask_rng_advance_kernel, dim3(1), dim3(32), 0, st, rng_state);
    SMK_CHECK_LAUNCH();
    return 0;
}
