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
project_kernel(const float* __restrict__ pts, const float* __restrict__ cam, int B, int L, int out_dim, float z_offset,
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
    if (out_dim == 3) {
        const float z = -__fmul_rn(s, p[2]);
        o[2] = z_offset != 0.f ? __fadd_rn(z, z_offset) : z;     // no add at 0: keeps -0 as -0
    }
}

// ---- masked sub-mesh: raster-space positions + vertex normals (util.py:30-62) ---------------------
__global__ void __launch_bounds__(128)
submesh_kernel(RenderDev d, const float* __restrict__ verts, const float* __restrict__ tverts, float raster_dz, int B,
               float* __restrict__ rv /*[B][NM][3]*/, float* __restrict__ normals /*[B][NM][3]*/) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int b = blockIdx.y;
    if (i >= d.NM) return;
    const float* vb = verts + (size_t)b * d.V * 3;
    const float* tv = tverts + ((size_t)b * d.V + d.mask_ids[i]) * 3;
    float* r = rv + ((size_t)b * d.NM + i) * 3;
    // renderer.py:144 (z + 10) and :172-173 (negate x,y) -> pytorch3d NDC, +X left, +Y up.  raster_dz = 10 - z_offset:
    // 10 for the face mask; 0 for the full head, whose tverts already carry the + 10 (tv[2] + 0 is tv[2]: never -0).
    r[0] = -tv[0]; r[1] = -tv[1]; r[2] = __fadd_rn(tv[2], raster_dz);
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

// =================================================================================================
// Backward: the gradient torch autograd takes through Renderer.forward (renderer.py:100-207,239-250,
// util.py:30-78) for verts and cam, with pytorch3d's rasterize_meshes backward for blur 0, K = 1, no
// perspective correction and no clipping (zbuf / dists carry no gradient: the reference uses neither).
// Four launches, no atomics, fixed-order sums:
//   render_bwd_face_kernel    one warp per face scans the face's conservative pixel range against the
//                             forward's pix_to_face: shading -> barycentrics -> raster-space x/y of the
//                             three corners, and the interpolated-normal gradient of the three corners.
//   render_bwd_normal_kernel  per sub-mesh vertex: gathers those over the CSR vertex -> face adjacency and
//                             backpropagates F.normalize(eps=1e-6) (util.py:62).
//   render_bwd_vertex_kernel  per mesh vertex: the cross products of util.py:52-57, the raster-space and
//                             transformed_vertices gradients through batch_orth_proj (util.py:64-78).
//   render_bwd_cam_kernel     per face: fixed-order reduction of the camera gradient.
constexpr int kFG = 15;                     // per-face gradient: x,y of 3 corners + normal of 3 corners

__device__ __forceinline__ void tri_raster_xy(const RenderDev& d, const float* vb, const int32_t* mask_ids,
                                              float s, float tx, float ty, int f, float* x, float* y) {
    // raster-space (pytorch3d NDC) x/y of the face's corners, bitwise as project_kernel + submesh_kernel
    for (int k = 0; k < 3; ++k) {
        const float* p = vb + (size_t)mask_ids[d.faces[(size_t)f * 3 + k]] * 3;
        x[k] = -__fmul_rn(s, __fadd_rn(p[0], tx));
        y[k] = __fmul_rn(s, __fadd_rn(p[1], ty));
    }
}

__global__ void __launch_bounds__(128)
render_bwd_face_kernel(RenderDev d, Lights lights, const float* __restrict__ verts, const float* __restrict__ cam,
                       const int64_t* __restrict__ p2f, const float* __restrict__ bary, const float* __restrict__ normals,
                       const float* __restrict__ g_rendered, int B, float* __restrict__ gface /*[B][F][15]*/) {
    const int lane = threadIdx.x & 31;
    const int f = blockIdx.x * 4 + (threadIdx.x >> 5), b = blockIdx.y;
    if (f >= d.F) return;
    float acc[kFG];
#pragma unroll
    for (int q = 0; q < kFG; ++q) acc[q] = 0.f;
    const float s = cam[b * 3], tx = cam[b * 3 + 1], ty = cam[b * 3 + 2];
    float x[3], y[3];
    tri_raster_xy(d, verts + (size_t)b * d.V * 3, d.mask_ids, s, tx, ty, f, x, y);
    const float xmin = fminf(x[0], fminf(x[1], x[2])), xmax = fmaxf(x[0], fmaxf(x[1], x[2]));
    const float ymin = fminf(y[0], fminf(y[1], y[2])), ymax = fmaxf(y[0], fmaxf(y[1], y[2]));
    const float hs = 0.5f * d.S;                 // the pixel range of tri_setup_kernel (a superset of the coverage)
    const float fx_lo = floorf((1.f - xmax) * hs - 0.5f) - 1.f, fx_hi = ceilf((1.f - xmin) * hs - 0.5f) + 1.f;
    const float fy_lo = floorf((1.f - ymax) * hs - 0.5f) - 1.f, fy_hi = ceilf((1.f - ymin) * hs - 0.5f) + 1.f;
    if (g_rendered && isfinite(xmin) && isfinite(xmax) && isfinite(ymin) && isfinite(ymax) &&
        fx_hi >= 0.f && fy_hi >= 0.f && fx_lo <= d.S - 1 && fy_lo <= d.S - 1) {
        const int xl = (int)fmaxf(fx_lo, 0.f), xh = (int)fminf(fx_hi, (float)(d.S - 1));
        const int yl = (int)fmaxf(fy_lo, 0.f), yh = (int)fminf(fy_hi, (float)(d.S - 1));
        const int nx = xh - xl + 1, npx = nx * (yh - yl + 1);
        const int64_t me = (int64_t)b * d.F + f;
        const size_t plane = (size_t)d.S * d.S;
        const float* nb = normals + (size_t)b * d.NM * 3;
        const int32_t* tri = d.faces + (size_t)f * 3;
        float n[3][3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int c = 0; c < 3; ++c) n[k][c] = nb[(size_t)tri[k] * 3 + c];
        // den = edge(v2; v0, v1) + 1e-8, as tri_setup_kernel
        const float den = __fadd_rn(edge_nf(x[2], y[2], x[0], y[0], x[1], y[1]), kEps);
        const float col = 180.0f / 255.0f;
        for (int q = lane; q < npx; q += 32) {
            const int xi = xl + q % nx, yi = yl + q / nx;
            const size_t pix = (size_t)yi * d.S + xi;
            if (p2f[(size_t)b * plane + pix] != me) continue;
            const float* gr = g_rendered + (size_t)b * 3 * plane + pix;
            const float G = (gr[0] + gr[plane]) + gr[2 * plane];          // the three channels are the same value
            const float* bw = bary + ((size_t)b * plane + pix) * 3;
            const float w[3] = {bw[0], bw[1], bw[2]};
            // forward recomputed in raster_tile_kernel's order (so the clamp masks match)
            const float alb = __fadd_rn(__fadd_rn(__fmul_rn(w[0], col), __fmul_rn(w[1], col)), __fmul_rn(w[2], col));
            float nn[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) nn[c] = __fadd_rn(__fadd_rn(__fmul_rn(w[0], n[0][c]), __fmul_rn(w[1], n[1][c])), __fmul_rn(w[2], n[2][c]));
            float sum = 0.f, gnn[3] = {0.f, 0.f, 0.f};
            bool pass[5];
#pragma unroll
            for (int l = 0; l < 5; ++l) {
                float dot = __fadd_rn(__fadd_rn(__fmul_rn(nn[0], lights.dir[l][0]), __fmul_rn(nn[1], lights.dir[l][1])),
                                      __fmul_rn(nn[2], lights.dir[l][2]));
                pass[l] = dot >= 0.f && dot <= 1.f;               // torch.clamp passes the gradient on [0, 1] inclusive
                dot = fminf(fmaxf(dot, 0.f), 1.f);
                sum = __fadd_rn(sum, __fmul_rn(dot, 1.7f));
            }
            // rendered = albedo * shading, shading = mean_l(1.7 clamp(n.l))           renderer.py:158-166,239-250
            const float g_alb = G * (sum / 5.0f);
            const float g_dot = G * alb * (1.7f / 5.0f);
#pragma unroll
            for (int l = 0; l < 5; ++l)
                if (pass[l])
#pragma unroll
                    for (int c = 0; c < 3; ++c) gnn[c] += g_dot * lights.dir[l][c];
            // interpolation (renderer.py:194-207): the albedo is the constant 180/255 at every corner
            float gw[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                gw[k] = g_alb * col + ((gnn[0] * n[k][0] + gnn[1] * n[k][1]) + gnn[2] * n[k][2]);
#pragma unroll
                for (int c = 0; c < 3; ++c) acc[6 + 3 * k + c] += w[k] * gnn[c];
            }
            // w_k = e_k / den with e0 = edge(p; v1, v2), e1 = edge(p; v2, v0), e2 = edge(p; v0, v1)
            // edge(p; a, b) = (px-ax)(by-ay) - (py-ay)(bx-ax): d/da = (py-by, bx-px), d/db = (ay-py, px-ax)
            const float xf = pix_to_ndc(d.S - 1 - xi, d.S), yf = pix_to_ndc(d.S - 1 - yi, d.S);
            const float ge[3] = {gw[0] / den, gw[1] / den, gw[2] / den};
            const float gden = -((gw[0] * w[0] + gw[1] * w[1]) + gw[2] * w[2]) / den;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int a = (k + 1) % 3, c = (k + 2) % 3;            // e_k = edge(p; v_a, v_c)
                acc[2 * a + 0] += ge[k] * (yf - y[c]);
                acc[2 * a + 1] += ge[k] * (x[c] - xf);
                acc[2 * c + 0] += ge[k] * (y[a] - yf);
                acc[2 * c + 1] += ge[k] * (xf - x[a]);
            }
            // den = edge(v2; v0, v1): d/dv2 = (y1-y0, x0-x1), d/dv0 = (y2-y1, x1-x2), d/dv1 = (y0-y2, x2-x0)
            acc[4] += gden * (y[1] - y[0]); acc[5] += gden * (x[0] - x[1]);
            acc[0] += gden * (y[2] - y[1]); acc[1] += gden * (x[1] - x[2]);
            acc[2] += gden * (y[0] - y[2]); acc[3] += gden * (x[2] - x[0]);
        }
    }
#pragma unroll
    for (int q = 0; q < kFG; ++q) {
        float v = acc[q];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        acc[q] = v;
    }
    if (lane < kFG) {
        float v = acc[0];
#pragma unroll
        for (int q = 1; q < kFG; ++q) if (lane == q) v = acc[q];
        gface[((size_t)b * d.F + f) * kFG + lane] = v;
    }
}

// raw (un-normalised) vertex normal of sub-mesh vertex i, as submesh_kernel
__device__ __forceinline__ void raw_normal(const RenderDev& d, const float* vb, int i, float* n) {
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
    n[0] = nx; n[1] = ny; n[2] = nz;
}

__global__ void __launch_bounds__(128)
render_bwd_normal_kernel(RenderDev d, const float* __restrict__ verts, const float* __restrict__ gface, int B,
                         float* __restrict__ graw /*[B][NM][3]*/, float* __restrict__ grv /*[B][NM][2]*/) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= d.NM) return;
    float gxy[2] = {0.f, 0.f}, gn[3] = {0.f, 0.f, 0.f};
    for (int e = d.adj_ptr[i]; e < d.adj_ptr[i + 1]; ++e) {
        const int code = d.adj[e], f = code >> 2, c = code & 3;
        const float* g = gface + ((size_t)b * d.F + f) * kFG;
        gxy[0] += g[2 * c]; gxy[1] += g[2 * c + 1];
        gn[0] += g[6 + 3 * c]; gn[1] += g[6 + 3 * c + 1]; gn[2] += g[6 + 3 * c + 2];
    }
    grv[((size_t)b * d.NM + i) * 2 + 0] = gxy[0];
    grv[((size_t)b * d.NM + i) * 2 + 1] = gxy[1];
    // y = x / max(||x||, 1e-6): g_x = g/den - x (x.g) / (den^2 ||x||) while ||x|| >= 1e-6
    float n[3];
    raw_normal(d, verts + (size_t)b * d.V * 3, i, n);
    const float len = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(n[0], n[0]), __fmul_rn(n[1], n[1])), __fmul_rn(n[2], n[2])));
    const float den = fmaxf(len, 1e-6f);
    const float xg = (n[0] * gn[0] + n[1] * gn[1]) + n[2] * gn[2];
    const float k = len >= 1e-6f ? xg / (den * den * len) : 0.f;
    float* o = graw + ((size_t)b * d.NM + i) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = gn[c] / den - n[c] * k;
}

__global__ void __launch_bounds__(128)
render_bwd_vertex_kernel(RenderDev d, const int32_t* __restrict__ inv_ptr, const int32_t* __restrict__ inv,
                         const float* __restrict__ verts, const float* __restrict__ cam, const float* __restrict__ graw,
                         const float* __restrict__ grv, const float* __restrict__ g_tverts, int B,
                         float* __restrict__ g_verts, float* __restrict__ gcam_v /*[B][V][3]*/) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (v >= d.V) return;
    const float* vb = verts + (size_t)b * d.V * 3;
    float gt[3] = {0.f, 0.f, 0.f}, gp[3] = {0.f, 0.f, 0.f};
    if (g_tverts) {
        const float* g = g_tverts + ((size_t)b * d.V + v) * 3;
        gt[0] = g[0]; gt[1] = g[1]; gt[2] = g[2];
    }
    for (int m = inv_ptr[v]; m < inv_ptr[v + 1]; ++m) {
        const int i = inv[m];
        // raster x, y = -tverts x, y (renderer.py:172-173); z only shifts and carries no gradient
        gt[0] -= grv[((size_t)b * d.NM + i) * 2 + 0];
        gt[1] -= grv[((size_t)b * d.NM + i) * 2 + 1];
        // util.py:52-57: corner c' adds cross(q1 - p, q2 - p) with p = c', q1 = c'+1, q2 = c'+2;
        // d cross(a, b) . G = da . (b x G) + db . (G x a)
        for (int e = d.adj_ptr[i]; e < d.adj_ptr[i + 1]; ++e) {
            const int code = d.adj[e], f = code >> 2, c = code & 3;
            const int32_t* tri = d.faces + (size_t)f * 3;
            float P[3][3], Gc[3][3];
#pragma unroll
            for (int k = 0; k < 3; ++k)
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    P[k][q] = vb[(size_t)d.mask_ids[tri[k]] * 3 + q];
                    Gc[k][q] = graw[((size_t)b * d.NM + tri[k]) * 3 + q];
                }
#pragma unroll
            for (int cp = 0; cp < 3; ++cp) {
                const int q1 = (cp + 1) % 3, q2 = (cp + 2) % 3;
                if (c != cp && c != q1 && c != q2) continue;
                float a[3], bb[3];
#pragma unroll
                for (int q = 0; q < 3; ++q) { a[q] = P[q1][q] - P[cp][q]; bb[q] = P[q2][q] - P[cp][q]; }
                const float* G = Gc[cp];
                const float ga[3] = {bb[1] * G[2] - bb[2] * G[1], bb[2] * G[0] - bb[0] * G[2], bb[0] * G[1] - bb[1] * G[0]};
                const float gb[3] = {G[1] * a[2] - G[2] * a[1], G[2] * a[0] - G[0] * a[2], G[0] * a[1] - G[1] * a[0]};
#pragma unroll
                for (int q = 0; q < 3; ++q)
                    gp[q] += c == cp ? -(ga[q] + gb[q]) : (c == q1 ? ga[q] : gb[q]);
            }
        }
    }
    // tverts = (s (x + tx), -s (y + ty), -s z)                                      util.py:64-78, renderer.py:102
    const float s = cam[b * 3], tx = cam[b * 3 + 1], ty = cam[b * 3 + 2];
    float* o = g_verts + ((size_t)b * d.V + v) * 3;
    o[0] = s * gt[0] + gp[0];
    o[1] = -s * gt[1] + gp[1];
    o[2] = -s * gt[2] + gp[2];
    float* gc = gcam_v + ((size_t)b * d.V + v) * 3;
    gc[0] = ((vb[v * 3] + tx) * gt[0] - (vb[v * 3 + 1] + ty) * gt[1]) - vb[v * 3 + 2] * gt[2];
    gc[1] = s * gt[0];
    gc[2] = -s * gt[1];
}

// out[b][k] = sum_i in[b][i][k], i < n, in a fixed order (strided per-thread sums, then a shared-memory tree)
__global__ void __launch_bounds__(256)
render_bwd_cam_kernel(const float* __restrict__ in, int n, float* __restrict__ out) {
    __shared__ float sR[3][256];
    const int b = blockIdx.x, tid = threadIdx.x;
    float a[3] = {0.f, 0.f, 0.f};
    for (int i = tid; i < n; i += 256)
#pragma unroll
        for (int k = 0; k < 3; ++k) a[k] += in[((size_t)b * n + i) * 3 + k];
#pragma unroll
    for (int k = 0; k < 3; ++k) sR[k][tid] = a[k];
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (tid < w)
#pragma unroll
            for (int k = 0; k < 3; ++k) sR[k][tid] += sR[k][tid + w];
        __syncthreads();
    }
    if (tid < 3) out[b * 3 + tid] = sR[tid][0];
}

// landmark projection backward (renderer.py:104-108): one CTA per face, x = s (px + tx), y = -s (py + ty);
// the camera gradient is summed over the points in a fixed order
__global__ void __launch_bounds__(128)
project_bwd_kernel(const float* __restrict__ pts, const float* __restrict__ cam, int L, const float* __restrict__ g_xy,
                   float* __restrict__ g_pts, float* __restrict__ g_cam) {
    __shared__ float sR[3][128];
    const int b = blockIdx.x, tid = threadIdx.x;
    const float s = cam[b * 3], tx = cam[b * 3 + 1], ty = cam[b * 3 + 2];
    float a[3] = {0.f, 0.f, 0.f};
    for (int l = tid; l < L; l += 128) {
        const size_t i = (size_t)b * L + l;
        const float* p = pts + i * 3;
        const float gx = g_xy[i * 2], gy = g_xy[i * 2 + 1];
        g_pts[i * 3] = s * gx; g_pts[i * 3 + 1] = -s * gy; g_pts[i * 3 + 2] = 0.f;
        a[0] += (p[0] + tx) * gx - (p[1] + ty) * gy;
        a[1] += s * gx;
        a[2] -= s * gy;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) sR[k][tid] = a[k];
    __syncthreads();
    for (int w = 64; w > 0; w >>= 1) {
        if (tid < w)
#pragma unroll
            for (int k = 0; k < 3; ++k) sR[k][tid] += sR[k][tid + w];
        __syncthreads();
    }
    if (tid < 3) g_cam[b * 3 + tid] = sR[tid][0];
}

}  // namespace

struct SmkRenderer {
    RenderDev d;
    Lights lights;
    float z_offset;        // added to the returned tverts' z (SmkRendererDesc::z_offset)
    int32_t* inv_ptr;      // [V+1] CSR mesh vertex -> sub-mesh ids (the inverse of mask_ids), for the backward
    int32_t* inv;          // [NM]
    smk::DeviceArena arena;
};

extern "C" int smk_renderer_create(const SmkRendererDesc* desc, SmkRenderer** out) {
    SMK_REQUIRE(desc && out && desc->mask_ids && desc->faces, "smk_renderer_create: null argument");
    SMK_REQUIRE(desc->image_size > 0 && desc->image_size % TILE_W == 0 && desc->image_size % TILE_H == 0 &&
                desc->image_size / TILE_H < 255, "smk_renderer_create: image_size must be a multiple of 32 (got %d)", desc->image_size);
    SMK_REQUIRE(desc->n_faces > 0 && desc->n_faces < 65536 && desc->n_faces % 4 == 0,
                "smk_renderer_create: n_faces must be in (0, 65536) and a multiple of 4 (got %d)", desc->n_faces);
    SMK_REQUIRE(desc->z_offset == 0.f || desc->z_offset == 10.f,            // the raster depth tv.z + (10 - z_offset) is z + 10
                "smk_renderer_create: z_offset must be 0 (face mask) or 10 (full head), got %g", (double)desc->z_offset);
    SmkRenderer* h = new SmkRenderer();
    RenderDev& d = h->d;
    d.V = desc->n_verts; d.NM = desc->n_mask; d.F = desc->n_faces; d.S = desc->image_size;
    h->z_offset = desc->z_offset;
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
    {   // backward: mesh vertex -> sub-mesh ids
        std::vector<int32_t> iptr(d.V + 1, 0), inv(std::max(d.NM, 1), 0);
        for (int i = 0; i < d.NM; ++i) iptr[desc->mask_ids[i] + 1]++;
        for (int v = 0; v < d.V; ++v) iptr[v + 1] += iptr[v];
        std::vector<int32_t> ifill(iptr.begin(), iptr.end() - 1);
        for (int i = 0; i < d.NM; ++i) inv[ifill[desc->mask_ids[i]]++] = i;
        if (e == cudaSuccess) e = h->arena.upload(iptr, &h->inv_ptr);
        if (e == cudaSuccess) e = h->arena.upload(inv, &h->inv);
    }
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
    SMK_LAUNCH(project_kernel, dim3(smk::cdiv((long)B * L, 256)), dim3(256), 0, (cudaStream_t)stream, pts, cam, B, L, 2, 0.f, out_xy);
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
    SMK_LAUNCH(project_kernel, dim3(smk::cdiv((long)B * d.V, 256)), dim3(256), 0, st, verts, cam, B, d.V, 3, h->z_offset, tverts);
    SMK_CHECK_LAUNCH();
    SMK_TAG("submesh_normals", 4.0 * B * (9.0 * d.NM) + 4.0 * (4.0 * d.F + 2.0 * d.NM), 30.0 * B * 3.0 * d.F, st);
    SMK_LAUNCH(submesh_kernel, dim3(dim3(smk::cdiv(d.NM, 128), B)), dim3(128), 0, st, d, verts, tverts, 10.0f - h->z_offset, B,
               rv, nrm);
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

// ---- backward ------------------------------------------------------------------------------------
extern "C" size_t smk_renderer_backward_workspace_bytes(const SmkRenderer* h, int B) {
    if (!h || B <= 0) return 0;
    const RenderDev& d = h->d;
    return smk::ws_round((size_t)B * d.F * kFG * 4) + smk::ws_round((size_t)B * d.NM * 3 * 4) +
           smk::ws_round((size_t)B * d.NM * 2 * 4) + smk::ws_round((size_t)B * d.V * 3 * 4);
}

extern "C" int smk_renderer_backward(const SmkRenderer* h, const float* verts, const float* cam, int B,
                                     const int64_t* pix_to_face, const float* bary, const float* normals,
                                     const float* g_rendered, const float* g_tverts, float* g_verts, float* g_cam,
                                     void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;
    SMK_REQUIRE(h && verts && cam && pix_to_face && bary && normals && g_verts && g_cam, "smk_renderer_backward: null argument");
    SMK_REQUIRE(B > 0, "smk_renderer_backward: negative batch");
    SMK_REQUIRE(ws && ws_bytes >= smk_renderer_backward_workspace_bytes(h, B), "smk_renderer_backward: workspace too small");
    const RenderDev& d = h->d;
    cudaStream_t st = (cudaStream_t)stream;
    smk::Workspace w(ws, ws_bytes);
    float* gface = w.take<float>((size_t)B * d.F * kFG);
    float* graw = w.take<float>((size_t)B * d.NM * 3);
    float* grv = w.take<float>((size_t)B * d.NM * 2);
    float* gcam_v = w.take<float>((size_t)B * d.V * 3);
    const double plane = (double)d.S * d.S;
    SMK_TAG("render_bwd_face", 4.0 * B * ((double)d.F * (kFG + 6) + 9.0 * d.NM + (g_rendered ? plane * (2 + 3 + 3) : 0.0)),
            g_rendered ? 120.0 * B * plane : 0.0, st);
    SMK_LAUNCH(render_bwd_face_kernel, dim3(smk::cdiv(d.F, 4), B), dim3(128), 0, st, d, h->lights, verts, cam,
               pix_to_face, bary, normals, g_rendered, B, gface);
    SMK_CHECK_LAUNCH();
    SMK_TAG("render_bwd_normal", 4.0 * B * ((double)d.F * kFG + 3.0 * d.NM + 5.0 * d.NM) + 4.0 * (4.0 * d.F + 2.0 * d.NM),
            B * (30.0 * 3.0 * d.F + 20.0 * d.NM), st);
    SMK_LAUNCH(render_bwd_normal_kernel, dim3(smk::cdiv(d.NM, 128), B), dim3(128), 0, st, d, verts, gface, B, graw, grv);
    SMK_CHECK_LAUNCH();
    SMK_TAG("render_bwd_vertex", 4.0 * B * (3.0 * d.V * (g_tverts ? 4 : 3) + 5.0 * d.NM + 6.0 * d.V) + 4.0 * (d.V + 1 + d.NM),
            B * (60.0 * 3.0 * d.F + 12.0 * d.V), st);
    SMK_LAUNCH(render_bwd_vertex_kernel, dim3(smk::cdiv(d.V, 128), B), dim3(128), 0, st, d, h->inv_ptr, h->inv, verts, cam,
               graw, grv, g_tverts, B, g_verts, gcam_v);
    SMK_CHECK_LAUNCH();
    SMK_TAG("render_bwd_cam", 4.0 * B * (3.0 * d.V + 3), 3.0 * B * d.V, st);
    SMK_LAUNCH(render_bwd_cam_kernel, dim3(B), dim3(256), 0, st, gcam_v, d.V, g_cam);
    SMK_CHECK_LAUNCH();
    return 0;
}

extern "C" int smk_project_points_backward(const float* pts, const float* cam, int B, int L, const float* g_xy,
                                           float* g_pts, float* g_cam, void* stream) {
    if (B == 0 || L == 0) return 0;            // empty batch: nothing to do (pointers may be null)
    SMK_REQUIRE(pts && cam && g_xy && g_pts && g_cam, "smk_project_points_backward: null argument");
    SMK_REQUIRE(B > 0 && L > 0, "smk_project_points_backward: negative size");
    SMK_TAG("project_points_bwd", 4.0 * B * (8.0 * L + 6), 12.0 * B * L, (cudaStream_t)stream);
    SMK_LAUNCH(project_bwd_kernel, dim3(B), dim3(128), 0, (cudaStream_t)stream, pts, cam, L, g_xy, g_pts, g_cam);
    SMK_CHECK_LAUNCH();
    return 0;
}
