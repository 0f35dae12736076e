// Mesh renderer on sm_90a: orthographic vertex stage, deterministic vertex normals, tiled
// edge-function rasteriser with shared-memory triangle binning, barycentric attribute interpolation
// and directional-light shading — one pass, no [B,F,3,6] attribute tensor, no atomics.
//
// Replaces Renderer.forward/render/rasterize/add_directionlight (reference src/renderer/renderer.py:
// 100-207,239-250), util.batch_orth_proj/vertex_normals/face_vertices (src/renderer/util.py) and the
// third-party pytorch3d `rasterize_meshes` call (renderer.py:185-193).
//
// Bit-exactness: coverage, face index and barycentrics follow the fp32 operation order of the naive
// pytorch3d rasteriser (see oracle/raster_ref.c) with explicitly un-fused multiplies/subtracts
// (this file is compiled with -fmad=false as well), so pix_to_face matches the CPU oracle exactly.
//
// This stage is integer/fp32-ALU + shared-memory work, not HBM- or tensor-bound: compulsory traffic is
// 60 KB of vertices in and 602 KB of image out per face.
#include "common.cuh"
#include <math.h>
#include <algorithm>

namespace {

constexpr int TILE_W = 32, TILE_H = 8;      // 224 = 7*32 = 28*8 -> 196 tiles per image, 128-byte row segments
constexpr int CHUNK = 64;                   // candidate triangles staged in shared memory at a time
constexpr int REC = 20;                     // floats per triangle record
constexpr float kEps = 1e-8f;

struct RenderDev {
    int V, NM, F, S;
    int32_t* mask_ids;     // [NM]
    int32_t* faces;        // [F][3] (sub-mesh numbering)
    int32_t* adj_ptr;      // [NM+1]  CSR vertex -> (face<<2 | corner), ordered like the reference's three
    int32_t* adj;          //         index_add_ passes (corner 1, then 2, then 0; faces ascending)
};

__device__ __forceinline__ float edge_nf(float px, float py, float ax, float ay, float bx, float by) {
    return __fsub_rn(__fmul_rn(__fsub_rn(px, ax), __fsub_rn(by, ay)), __fmul_rn(__fsub_rn(py, ay), __fsub_rn(bx, ax)));
}

__device__ __forceinline__ float pix_to_ndc(int i, int S) {
    return __fadd_rn(-1.0f, __fdiv_rn(__fadd_rn(__fmul_rn(2.0f, (float)i), 1.0f), (float)S));
}

// ---- vertex stage: util.batch_orth_proj + sign flips (renderer.py:101-102) ------------------------
__global__ void __launch_bounds__(256)
project_kernel(const float* __restrict__ pts, const float* __restrict__ cam, int B, int L, int out_dim,
               float* __restrict__ out) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * L) return;
    int b = (int)(i / L);
    float s = cam[b * 3], tx = cam[b * 3 + 1], ty = cam[b * 3 + 2];
    const float* p = pts + i * 3;
    float x = __fmul_rn(s, __fadd_rn(p[0], tx));
    float y = -__fmul_rn(s, __fadd_rn(p[1], ty));
    float* o = out + i * out_dim;
    o[0] = x; o[1] = y;
    if (out_dim == 3) o[2] = -__fmul_rn(s, p[2]);
}

// ---- masked sub-mesh: raster-space positions + vertex normals (util.py:30-62) ---------------------
__global__ void __launch_bounds__(128)
submesh_kernel(RenderDev d, const float* __restrict__ verts, const float* __restrict__ tverts, int B,
               float* __restrict__ rv /*[B][NM][3]*/, float* __restrict__ normals /*[B][NM][3]*/) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int b = blockIdx.y;
    if (i >= d.NM) return;
    const float* vb = verts + (size_t)b * d.V * 3;
    const float* tv = tverts + ((size_t)b * d.V + d.mask_ids[i]) * 3;
    float* r = rv + ((size_t)b * d.NM + i) * 3;
    // renderer.py:144 (z += 10) and :172-173 (negate x,y) -> pytorch3d NDC, +X left, +Y up
    r[0] = -tv[0]; r[1] = -tv[1]; r[2] = __fadd_rn(tv[2], 10.0f);
    float nx = 0.f, ny = 0.f, nz = 0.f;
    for (int e = d.adj_ptr[i]; e < d.adj_ptr[i + 1]; ++e) {
        int code = d.adj[e], f = code >> 2, c = code & 3;
        const int32_t* tri = d.faces + (size_t)f * 3;
        const float* p = vb + (size_t)d.mask_ids[tri[c]] * 3;
        const float* q1 = vb + (size_t)d.mask_ids[tri[(c + 1) % 3]] * 3;
        const float* q2 = vb + (size_t)d.mask_ids[tri[(c + 2) % 3]] * 3;
        float ax = q1[0] - p[0], ay = q1[1] - p[1], az = q1[2] - p[2];
        float bx = q2[0] - p[0], by = q2[1] - p[1], bz = q2[2] - p[2];
        nx += __fsub_rn(__fmul_rn(ay, bz), __fmul_rn(az, by));
        ny += __fsub_rn(__fmul_rn(az, bx), __fmul_rn(ax, bz));
        nz += __fsub_rn(__fmul_rn(ax, by), __fmul_rn(ay, bx));
    }
    float len = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
    float den = fmaxf(len, 1e-6f);                         // F.normalize(eps=1e-6)
    float* n = normals + ((size_t)b * d.NM + i) * 3;
    n[0] = __fdiv_rn(nx, den); n[1] = __fdiv_rn(ny, den); n[2] = __fdiv_rn(nz, den);
}

// ---- triangle setup -------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
tri_setup_kernel(RenderDev d, const float* __restrict__ rv, int B, float* __restrict__ recs /*[B][F][REC]*/,
                 uint32_t* __restrict__ ranges /*[B][F]*/) {
    int f = blockIdx.x * blockDim.x + threadIdx.x;
    int b = blockIdx.y;
    if (f >= d.F) return;
    const int32_t* tri = d.faces + (size_t)f * 3;
    const float* base = rv + (size_t)b * d.NM * 3;
    const float* p0 = base + (size_t)tri[0] * 3; const float* p1 = base + (size_t)tri[1] * 3; const float* p2 = base + (size_t)tri[2] * 3;
    float x0 = p0[0], y0 = p0[1], z0 = p0[2], x1 = p1[0], y1 = p1[1], z1 = p1[2], x2 = p2[0], y2 = p2[1], z2 = p2[2];
    float area = edge_nf(x0, y0, x1, y1, x2, y2);
    float xmin = fminf(x0, fminf(x1, x2)), xmax = fmaxf(x0, fmaxf(x1, x2));
    float ymin = fminf(y0, fminf(y1, y2)), ymax = fmaxf(y0, fmaxf(y1, y2));
    float zmax = fmaxf(z0, fmaxf(z1, z2));
    float* r = recs + ((size_t)b * d.F + f) * REC;
    float4* r4 = reinterpret_cast<float4*>(r);
    r4[0] = make_float4(x0, y0, x1, y1);
    r4[1] = make_float4(x2, y2, __fsub_rn(y2, y1), __fsub_rn(x2, x1));
    r4[2] = make_float4(__fsub_rn(y0, y2), __fsub_rn(x0, x2), __fsub_rn(y1, y0), __fsub_rn(x1, x0));
    r4[3] = make_float4(z0, z1, z2, __fadd_rn(edge_nf(x2, y2, x0, y0, x1, y1), kEps));
    r4[4] = make_float4(xmin, xmax, ymin, ymax);
    // conservative tile range; pixel xi samples xf = 1 - (2 xi + 1)/S  <=>  xi = (1 - xf) S/2 - 1/2
    bool valid = !(area <= kEps && area >= -kEps) && !(zmax < 0.f) &&
                 isfinite(xmin) && isfinite(xmax) && isfinite(ymin) && isfinite(ymax);
    const float hs = 0.5f * d.S;
    float fx_lo = floorf((1.f - xmax) * hs - 0.5f) - 1.f, fx_hi = ceilf((1.f - xmin) * hs - 0.5f) + 1.f;
    float fy_lo = floorf((1.f - ymax) * hs - 0.5f) - 1.f, fy_hi = ceilf((1.f - ymin) * hs - 0.5f) + 1.f;
    uint32_t code = 0x000000FFu;                         // empty: tx0 = 255 > tx1 = 0
    if (valid && fx_hi >= 0.f && fy_hi >= 0.f && fx_lo <= d.S - 1 && fy_lo <= d.S - 1) {
        int xl = (int)fmaxf(fx_lo, 0.f), xh = (int)fminf(fx_hi, (float)(d.S - 1));
        int yl = (int)fmaxf(fy_lo, 0.f), yh = (int)fminf(fy_hi, (float)(d.S - 1));
        code = (uint32_t)(xl / TILE_W) | ((uint32_t)(xh / TILE_W) << 8) | ((uint32_t)(yl / TILE_H) << 16) | ((uint32_t)(yh / TILE_H) << 24);
    }
    ranges[(size_t)b * d.F + f] = code;
}

// ---- tile rasteriser + shading ----------------------------------------------------------------------
struct Lights { float dir[5][3]; };

__global__ void __launch_bounds__(TILE_W * TILE_H)
raster_tile_kernel(RenderDev d, const float* __restrict__ recs, const uint32_t* __restrict__ ranges,
                   const float* __restrict__ normals, Lights lights, int B,
                   float* __restrict__ rendered, int64_t* __restrict__ p2f, float* __restrict__ bary,
                   float* __restrict__ zbuf) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* s_tri = reinterpret_cast<float*>(smem_raw);                       // [CHUNK][REC]
    uint16_t* s_cand = reinterpret_cast<uint16_t*>(s_tri + CHUNK * REC);     // [F]
    __shared__ int s_count;
    const int tid = threadIdx.y * TILE_W + threadIdx.x;
    const int nthr = TILE_W * TILE_H;
    const int b = blockIdx.z;
    const uint32_t tx = blockIdx.x, ty = blockIdx.y;
    if (tid == 0) s_count = 0;
    __syncthreads();
    // -- bin: compact the ids of triangles whose conservative tile range covers this tile
    //    (4 packed ranges per thread per pass: one 16-byte load, one shared atomic per warp)
    const uint4* rg4 = reinterpret_cast<const uint4*>(ranges + (size_t)b * d.F);
    const int F4 = d.F >> 2;                                  // F % 4 == 0 is checked at create time
    for (int base0 = 0; base0 < F4; base0 += 4 * nthr) {
      uint4 pre[4];                                           // four independent 16-byte loads in flight: one L2 round trip per 4 passes
#pragma unroll
      for (int u = 0; u < 4; ++u) {
          const int j4 = base0 + u * nthr + tid;
          pre[u] = j4 < F4 ? __ldg(rg4 + j4) : make_uint4(0xFFu, 0xFFu, 0xFFu, 0xFFu);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i4 = base0 + u * nthr + tid;
        const uint32_t c[4] = {pre[u].x, pre[u].y, pre[u].z, pre[u].w};
        unsigned hits = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            bool hit = (c[k] & 0xFF) <= tx && tx <= ((c[k] >> 8) & 0xFF) && ((c[k] >> 16) & 0xFF) <= ty && ty <= (c[k] >> 24);
            hits |= (hit ? 1u : 0u) << k;
        }
        if (__ballot_sync(0xffffffffu, hits != 0) == 0) continue;      // warp-uniform: a tile sees ~1 % of the faces
        const int lane = tid & 31;
        const int mine = __popc(hits);
        int incl = mine;                                      // inclusive warp scan of the per-lane hit counts
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        int wbase = 0;
        if (lane == 31 && total) wbase = atomicAdd(&s_count, total);
        wbase = __shfl_sync(0xffffffffu, wbase, 31);
        int pos = wbase + incl - mine;
#pragma unroll
        for (int k = 0; k < 4; ++k) if (hits & (1u << k)) s_cand[pos++] = (uint16_t)(i4 * 4 + k);
      }
    }
    __syncthreads();
    const int ncand = s_count;
    const int xi = tx * TILE_W + threadIdx.x, yi = ty * TILE_H + threadIdx.y;
    const float xf = pix_to_ndc(d.S - 1 - xi, d.S), yf = pix_to_ndc(d.S - 1 - yi, d.S);
    int best_f = -1;
    float best_z = 0.f, bw0 = 0.f, bw1 = 0.f, bw2 = 0.f;
    const float* rb = recs + (size_t)b * d.F * REC;
    for (int c0 = 0; c0 < ncand; c0 += CHUNK) {
        int n = min(CHUNK, ncand - c0);
        __syncthreads();
        for (int i = tid; i < n * (REC / 4); i += nthr) {
            int t = i / (REC / 4), q = i % (REC / 4);
            reinterpret_cast<float4*>(s_tri)[t * (REC / 4) + q] =
                reinterpret_cast<const float4*>(rb + (size_t)s_cand[c0 + t] * REC)[q];
        }
        __syncthreads();
        // A warp is one pixel row of the tile (same yf in every lane): lane l first tests candidates l and
        // l+32 against the row's y and the row's x-extent, the ballots become the warp's work list, and
        // only the survivors (about a third) reach the per-pixel tests.
        const float xf_hi = pix_to_ndc(d.S - 1 - (int)(tx * TILE_W), d.S);                 // lane 0 sees the largest xf
        const float xf_lo = pix_to_ndc(d.S - 1 - (int)(tx * TILE_W + TILE_W - 1), d.S);
        const int lane = tid & 31;
        unsigned long long live = 0ull;
#pragma unroll
        for (int hseg = 0; hseg < CHUNK / 32; ++hseg) {
            const int t = hseg * 32 + lane;
            bool ok = false;
            if (t < n) {
                const float4 bb = *reinterpret_cast<const float4*>(s_tri + t * REC + 16);    // xmin, xmax, ymin, ymax
                ok = !(yf > bb.w || yf < bb.z) && !(xf_lo > bb.y || xf_hi < bb.x);
            }
            live |= (unsigned long long)__ballot_sync(0xffffffffu, ok) << (32 * hseg);
        }
        while (live) {
            const int t = __ffsll((long long)live) - 1;
            live &= live - 1;
            const float* r = s_tri + t * REC;
            if (xf > r[17] || xf < r[16]) continue;                                  // outside bbox in x (y was tested per row)
            float e0 = __fsub_rn(__fmul_rn(__fsub_rn(xf, r[2]), r[6]), __fmul_rn(__fsub_rn(yf, r[3]), r[7]));    // edge(p; v1, v2)
            float e1 = __fsub_rn(__fmul_rn(__fsub_rn(xf, r[4]), r[8]), __fmul_rn(__fsub_rn(yf, r[5]), r[9]));    // edge(p; v2, v0)
            float e2 = __fsub_rn(__fmul_rn(__fsub_rn(xf, r[0]), r[10]), __fmul_rn(__fsub_rn(yf, r[1]), r[11]));  // edge(p; v0, v1)
            float den = r[15];
            // sign pre-filter (exact: a quotient with the wrong sign or a zero numerator is never > 0)
            bool pos = den > 0.f;
            if (pos ? !(e0 > 0.f && e1 > 0.f && e2 > 0.f) : !(e0 < 0.f && e1 < 0.f && e2 < 0.f)) continue;
            float w0 = __fdiv_rn(e0, den), w1 = __fdiv_rn(e1, den), w2 = __fdiv_rn(e2, den);
            if (!(w0 > 0.f && w1 > 0.f && w2 > 0.f)) continue;
            float pz = __fadd_rn(__fadd_rn(__fmul_rn(w0, r[12]), __fmul_rn(w1, r[13])), __fmul_rn(w2, r[14]));
            if (pz < 0.f) continue;
            int f = s_cand[c0 + t];
            if (best_f < 0 || pz < best_z || (pz == best_z && f < best_f)) {
                best_f = f; best_z = pz; bw0 = w0; bw1 = w1; bw2 = w2;
            }
        }
    }
    // -- interpolate + shade (renderer.py:194-207, 158-166, 239-250)
    float val = 0.f;
    if (best_f >= 0) {
        const int32_t* tri = d.faces + (size_t)best_f * 3;
        const float* nb = normals + (size_t)b * d.NM * 3;
        const float* n0 = nb + (size_t)tri[0] * 3; const float* n1 = nb + (size_t)tri[1] * 3; const float* n2 = nb + (size_t)tri[2] * 3;
        const float col = 180.0f / 255.0f;
        float alb = __fadd_rn(__fadd_rn(__fmul_rn(bw0, col), __fmul_rn(bw1, col)), __fmul_rn(bw2, col));
        float nn[3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
            nn[k] = __fadd_rn(__fadd_rn(__fmul_rn(bw0, n0[k]), __fmul_rn(bw1, n1[k])), __fmul_rn(bw2, n2[k]));
        float sum = 0.f;
#pragma unroll
        for (int l = 0; l < 5; ++l) {
            float dot = __fadd_rn(__fadd_rn(__fmul_rn(nn[0], lights.dir[l][0]), __fmul_rn(nn[1], lights.dir[l][1])),
                                  __fmul_rn(nn[2], lights.dir[l][2]));
            dot = fminf(fmaxf(dot, 0.f), 1.f);
            sum = __fadd_rn(sum, __fmul_rn(dot, 1.7f));
        }
        val = __fmul_rn(alb, __fdiv_rn(sum, 5.0f));
    }
    const size_t plane = (size_t)d.S * d.S;
    const size_t pix = (size_t)yi * d.S + xi;
    float* o = rendered + (size_t)b * 3 * plane + pix;
    o[0] = val; o[plane] = val; o[2 * plane] = val;
    if (p2f) p2f[(size_t)b * plane + pix] = best_f >= 0 ? (int64_t)b * d.F + best_f : (int64_t)-1;
    if (zbuf) zbuf[(size_t)b * plane + pix] = best_f >= 0 ? best_z : -1.f;
    if (bary) {
        float* bo = bary + ((size_t)b * plane + pix) * 3;
        bo[0] = best_f >= 0 ? bw0 : -1.f; bo[1] = best_f >= 0 ? bw1 : -1.f; bo[2] = best_f >= 0 ? bw2 : -1.f;
    }
}

}  // namespace

struct SmkRenderer {
    RenderDev d;
    Lights lights;
    smk::DeviceArena arena;
};

extern "C" int smk_renderer_create(const SmkRendererDesc* desc, SmkRenderer** out) {
    SMK_REQUIRE(desc && out && desc->mask_ids && desc->faces, "smk_renderer_create: null argument");
    SMK_REQUIRE(desc->image_size > 0 && desc->image_size % TILE_W == 0 && desc->image_size % TILE_H == 0 &&
                desc->image_size / TILE_H < 255, "smk_renderer_create: image_size must be a multiple of 32 (got %d)", desc->image_size);
    SMK_REQUIRE(desc->n_faces > 0 && desc->n_faces < 65536 && desc->n_faces % 4 == 0,
                "smk_renderer_create: n_faces must be in (0, 65536) and a multiple of 4 (got %d)", desc->n_faces);
    SmkRenderer* h = new SmkRenderer();
    RenderDev& d = h->d;
    d.V = desc->n_verts; d.NM = desc->n_mask; d.F = desc->n_faces; d.S = desc->image_size;
    for (int i = 0; i < d.NM; ++i)
        if (desc->mask_ids[i] < 0 || desc->mask_ids[i] >= d.V) { delete h; smk::set_error("smk_renderer_create: mask id out of range"); return -1; }
    for (int i = 0; i < d.F * 3; ++i)
        if (desc->faces[i] < 0 || desc->faces[i] >= d.NM) { delete h; smk::set_error("smk_renderer_create: face index out of range"); return -1; }
    // CSR adjacency in the order of the reference's three index_add_ passes (util.py:52-57):
    // all faces' corner 1, then corner 2, then corner 0.
    std::vector<int32_t> ptr(d.NM + 1, 0), adj((size_t)d.F * 3);
    for (int i = 0; i < d.F * 3; ++i) ptr[desc->faces[i] + 1]++;
    for (int i = 0; i < d.NM; ++i) ptr[i + 1] += ptr[i];
    std::vector<int32_t> fill(ptr.begin(), ptr.end() - 1);
    const int order[3] = {1, 2, 0};
    for (int pass = 0; pass < 3; ++pass)
        for (int f = 0; f < d.F; ++f) {
            int c = order[pass];
            adj[fill[desc->faces[f * 3 + c]]++] = (f << 2) | c;
        }
    cudaError_t e = h->arena.upload(desc->mask_ids, (size_t)d.NM, &d.mask_ids);
    if (e == cudaSuccess) e = h->arena.upload(desc->faces, (size_t)d.F * 3, &d.faces);
    if (e == cudaSuccess) e = h->arena.upload(ptr, &d.adj_ptr);
    if (e == cudaSuccess) e = h->arena.upload(adj, &d.adj);
    if (e != cudaSuccess) { smk::set_error("smk_renderer_create: upload failed: %s", cudaGetErrorString(e)); delete h; return (int)e; }
    // light directions, F.normalize(dir) = dir / max(||dir||, 1e-12)      renderer.py:127-135,247
    const float dirs[5][3] = {{-1, 1, 1}, {1, 1, 1}, {-1, -1, 1}, {1, -1, 1}, {0, 0, 1}};
    for (int l = 0; l < 5; ++l) {
        float n = sqrtf(dirs[l][0] * dirs[l][0] + dirs[l][1] * dirs[l][1] + dirs[l][2] * dirs[l][2]);
        n = std::max(n, 1e-12f);
        for (int k = 0; k < 3; ++k) h->lights.dir[l][k] = dirs[l][k] / n;
    }
    *out = h;
    return 0;
}

extern "C" void smk_renderer_destroy(SmkRenderer* h) { delete h; }

extern "C" size_t smk_renderer_workspace_bytes(const SmkRenderer* h, int B) {
    const RenderDev& d = h->d;
    return smk::ws_round((size_t)B * d.NM * 3 * 4) * 2 + smk::ws_round((size_t)B * d.F * REC * 4) + smk::ws_round((size_t)B * d.F * 4);
}

extern "C" int smk_project_points(const float* pts, const float* cam, int B, int L, float* out_xy, void* stream) {
    SMK_REQUIRE(pts && cam && out_xy, "smk_project_points: null argument");
    if (B <= 0 || L <= 0) return 0;
    SMK_TAG("project_points", 4.0 * B * (5.0 * L + 3), 4.0 * B * L, (cudaStream_t)stream);
    SMK_LAUNCH(project_kernel, dim3(smk::cdiv((long)B * L, 256)), dim3(256), 0, (cudaStream_t)stream, pts, cam, B, L, 2, out_xy);
    SMK_CHECK_LAUNCH();
    return 0;
}

extern "C" int smk_renderer_forward(const SmkRenderer* h, const float* verts, const float* cam, int B,
                                    float* rendered, float* tverts, int64_t* pix_to_face, float* bary, float* zbuf,
                                    float* normals_out, void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;                      // empty batch: nothing to do (pointers may be null)
    SMK_REQUIRE(h && verts && cam && rendered && tverts, "smk_renderer_forward: null argument");
    SMK_REQUIRE(B > 0, "smk_renderer_forward: negative batch");
    SMK_REQUIRE(ws && ws_bytes >= smk_renderer_workspace_bytes(h, B), "smk_renderer_forward: workspace too small");
    const RenderDev& d = h->d;
    cudaStream_t st = (cudaStream_t)stream;
    smk::Workspace w(ws, ws_bytes);
    float* rv = w.take<float>((size_t)B * d.NM * 3);
    float* nrm_ws = w.take<float>((size_t)B * d.NM * 3);
    float* recs = w.take<float>((size_t)B * d.F * REC);
    uint32_t* ranges = w.take<uint32_t>((size_t)B * d.F);
    float* nrm = normals_out ? normals_out : nrm_ws;
    SMK_TAG("project_verts", 4.0 * B * (6.0 * d.V + 3), 5.0 * B * d.V, st);
    SMK_LAUNCH(project_kernel, dim3(smk::cdiv((long)B * d.V, 256)), dim3(256), 0, st, verts, cam, B, d.V, 3, tverts);
    SMK_CHECK_LAUNCH();
    SMK_TAG("submesh_normals", 4.0 * B * (9.0 * d.NM) + 4.0 * (4.0 * d.F + 2.0 * d.NM), 30.0 * B * 3.0 * d.F, st);
    SMK_LAUNCH(submesh_kernel, dim3(dim3(smk::cdiv(d.NM, 128), B)), dim3(128), 0, st, d, verts, tverts, B, rv, nrm);
    SMK_CHECK_LAUNCH();
    SMK_TAG("tri_setup", 4.0 * B * (3.0 * d.NM + (double)d.F * (REC + 1)) + 12.0 * d.F, 40.0 * B * d.F, st);
    SMK_LAUNCH(tri_setup_kernel, dim3(dim3(smk::cdiv(d.F, 128), B)), dim3(128), 0, st, d, rv, B, recs, ranges);
    SMK_CHECK_LAUNCH();
    size_t smem = (size_t)CHUNK * REC * 4 + (((size_t)d.F * 2 + 15) & ~size_t(15));
    dim3 grid(d.S / TILE_W, d.S / TILE_H, B);
    SMK_TAG("raster_tile", 4.0 * B * ((double)d.F * (REC + 1) + 3.0 * d.NM + (double)d.S * d.S * (3 + (pix_to_face ? 2 : 0) + (bary ? 3 : 0) + (zbuf ? 1 : 0))), 0.0, st);
    SMK_LAUNCH(raster_tile_kernel, dim3(grid), dim3(dim3(TILE_W, TILE_H)), smem, st, d, recs, ranges, nrm, h->lights, B, rendered, pix_to_face, bary, zbuf);
    SMK_CHECK_LAUNCH();
    return 0;
}
