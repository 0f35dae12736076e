// FLAME forward on sm_90a: blendshapes + pose correctives + linear blend skinning + eyelids + landmarks.
//
// Replaces FLAME.forward (reference src/FLAME/FLAME.py:232-315) and lbs() (src/FLAME/lbs.py:140-227).
// Three launches per batch, all fp32 FMA (this stage is memory/latency bound; tensor cores would
// cost the 1e-4 vertex tolerance and gain nothing):
//   flame_pose_kernel   one CTA per face: joints J = J0 + JS*beta (the joint regressor pre-contracted
//                       with shapedirs at create time), Rodrigues (lbs.py:274-305), kinematic chain
//                       (lbs.py:321-378) in registers, pose feature (lbs.py:197), contour-LUT row
//                       (FLAME.py:117-159).
//   flame_verts_kernel  CTA = 32 vertices x 4 k-slices, BT faces per thread in registers; each warp
//                       streams its quarter of the transposed shapedirs [350][3V] and posedirs
//                       (384 contiguous bytes per load), partial sums meet in shared memory, then
//                       the vertices are skinned with the 5 joint transforms held in shared memory
//                       and the eyelid offsets are added (FLAME.py:284-286).
//   flame_landmarks_kernel  241 barycentric gathers per face (lbs.py:101-137).
#include "common.cuh"
#include <math.h>

namespace {

constexpr int kJ = 5;          // joints; parents = [-1,0,1,1,1]  (FLAME.py:76-77)
constexpr int kPF = 36;        // (J-1)*9 pose-corrective features

struct FlameDev {
    int V, F, L, Mp;                       // Mp = 3V rounded up to a multiple of 4
    float* sdt;        // [L][Mp]   shapedirs transposed: sdt[l][3v+k] = shapedirs[v][k][l]
    float* pdt;        // [36][Mp]  posedirs (already [P][3V] in the reference), row-padded
    float* vt;         // [Mp]      v_template
    float* wt;         // [5][V]    lbs weights transposed
    float* leye;       // [Mp]
    float* reye;       // [Mp]
    float* js;         // [15][L]   J_regressor * shapedirs
    float* j0;         // [15]      J_regressor * v_template
    int32_t* faces;    // [F][3]
    int n_static, n_dyn_rows, n_dyn, n_full, n_mp;
    int32_t *static_faces, *dyn_faces, *full_faces, *mp_faces;
    float *static_bary, *dyn_bary, *full_bary, *mp_bary;
};

// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void rodrigues(const float* r, float* R) {
    // lbs.py:289-304: eps is added inside the norm only; R = I + sin*K + (1-cos)*K*K.
    float ax = r[0] + 1e-8f, ay = r[1] + 1e-8f, az = r[2] + 1e-8f;
    float angle = sqrtf(ax * ax + ay * ay + az * az);
    float rx = r[0] / angle, ry = r[1] / angle, rz = r[2] / angle;
    float s = sinf(angle), c = cosf(angle);
    float K[9] = {0.f, -rz, ry, rz, 0.f, -rx, -ry, rx, 0.f};
    float KK[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            KK[i * 3 + j] = K[i * 3 + 0] * K[0 * 3 + j] + K[i * 3 + 1] * K[1 * 3 + j] + K[i * 3 + 2] * K[2 * 3 + j];
    float omc = 1.f - c;
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = ((i % 4 == 0) ? 1.f : 0.f) + s * K[i] + omc * KK[i];
}

// G = P * [R | t]  (3x4 affine; bottom row 0 0 0 1 implied)
__device__ __forceinline__ void affine_mul(const float* P, const float* R, const float* t, float* G) {
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j)
            G[i * 4 + j] = P[i * 4 + 0] * R[0 * 3 + j] + P[i * 4 + 1] * R[1 * 3 + j] + P[i * 4 + 2] * R[2 * 3 + j];
        G[i * 4 + 3] = P[i * 4 + 0] * t[0] + P[i * 4 + 1] * t[1] + P[i * 4 + 2] * t[2] + P[i * 4 + 3];
    }
}

__global__ void __launch_bounds__(128)
flame_pose_kernel(FlameDev d, const float* __restrict__ betas, const float* __restrict__ full_pose, int B,
                  float* __restrict__ A_out /*[B][60]*/, float* __restrict__ pf_out /*[B][36]*/,
                  float* __restrict__ joints_out /*[B][5][3] or null*/, int32_t* __restrict__ dyn_out /*[B]*/) {
    __shared__ float sJ[15];
    __shared__ float sR[kJ][9];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* beta = betas + (size_t)b * d.L;
    // J = J0 + JS * beta : 15 dot products of length L, one warp per row (lbs.py:188 pre-contracted)
    for (int row = warp; row < 15; row += 4) {
        const float* js = d.js + (size_t)row * d.L;
        float acc = 0.f;
        for (int l = lane; l < d.L; l += 32) acc = fmaf(js[l], beta[l], acc);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) sJ[row] = d.j0[row] + acc;
    }
    if (tid < kJ) rodrigues(full_pose + (size_t)b * 15 + tid * 3, sR[tid]);
    __syncthreads();
    if (tid < kPF) {                 // pose_feature = (R[1:] - I).view(36)      lbs.py:197
        int j = 1 + tid / 9, e = tid % 9;
        pf_out[(size_t)b * kPF + tid] = sR[j][e] - ((e % 4 == 0) ? 1.f : 0.f);
    }
    if (tid == 0) {
        // kinematic chain, parents [-1,0,1,1,1]                                   lbs.py:345-363
        float G[kJ][12];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
#pragma unroll
            for (int j = 0; j < 3; ++j) G[0][i * 4 + j] = sR[0][i * 3 + j];
            G[0][i * 4 + 3] = sJ[i];
        }
        float rel[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) rel[k] = sJ[3 + k] - sJ[k];
        affine_mul(G[0], sR[1], rel, G[1]);
#pragma unroll
        for (int j = 2; j < kJ; ++j) {
#pragma unroll
            for (int k = 0; k < 3; ++k) rel[k] = sJ[3 * j + k] - sJ[3 + k];
            affine_mul(G[1], sR[j], rel, G[j]);
        }
        // A = G - pad(G * [J;0])                                                  lbs.py:373-376
        float* A = A_out + (size_t)b * 60;
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                float corr = G[j][i * 4 + 0] * sJ[3 * j] + G[j][i * 4 + 1] * sJ[3 * j + 1] + G[j][i * 4 + 2] * sJ[3 * j + 2];
                A[j * 12 + i * 4 + 0] = G[j][i * 4 + 0];
                A[j * 12 + i * 4 + 1] = G[j][i * 4 + 1];
                A[j * 12 + i * 4 + 2] = G[j][i * 4 + 2];
                A[j * 12 + i * 4 + 3] = G[j][i * 4 + 3] - corr;
                if (joints_out) joints_out[((size_t)b * kJ + j) * 3 + i] = G[j][i * 4 + 3];
            }
        }
        // dynamic contour row (FLAME.py:133-153): rel = R_global * R_neck, yaw about y
        float M[9];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j)
                M[i * 3 + j] = sR[0][i * 3 + 0] * sR[1][0 * 3 + j] + sR[0][i * 3 + 1] * sR[1][1 * 3 + j] + sR[0][i * 3 + 2] * sR[1][2 * 3 + j];
        float sy = sqrtf(M[0] * M[0] + M[3] * M[3]);
        float yaw = atan2f(-M[6], sy);
        float deg = (yaw * 180.0f) / 3.14159265358979323846f;
        deg = fminf(deg, 39.f);
        int y = (int)rintf(deg);                          // torch.round = half-to-even
        if (y < 0) y = (y < -39) ? 78 : (39 - y);
        if (dyn_out) dyn_out[b] = y;
    }
}

// -------------------------------------------------------------------------------------------------
template <int BT>
__global__ void __launch_bounds__(128)
flame_verts_kernel(FlameDev d, const float* __restrict__ betas, const float* __restrict__ eyelid,
                   const float* __restrict__ A_in, const float* __restrict__ pf_in, int B,
                   float* __restrict__ verts) {
    extern __shared__ float smem[];
    float* sB = smem;                       // [L][BT]   (beta for the BT faces adjacent -> one LDS.128 per l)
    float* sP = sB + (size_t)d.L * BT;      // [36][BT]
    float* sA = sP + kPF * BT;              // [BT][60]
    float* sE = sA + BT * 60;               // [BT][2]
    const int b0 = blockIdx.y * BT;
    const int tid = threadIdx.x;
    for (int i = tid; i < d.L * BT; i += 128) {
        int l = i / BT, t = i % BT;
        int b = min(b0 + t, B - 1);
        sB[i] = betas[(size_t)b * d.L + l];
    }
    for (int i = tid; i < kPF * BT; i += 128) {
        int p = i / BT, t = i % BT;
        sP[i] = pf_in[(size_t)min(b0 + t, B - 1) * kPF + p];
    }
    for (int i = tid; i < BT * 60; i += 128) sA[i] = A_in[(size_t)min(b0 + i / 60, B - 1) * 60 + i % 60];
    if (tid < BT * 2) sE[tid] = eyelid ? eyelid[(size_t)min(b0 + tid / 2, B - 1) * 2 + (tid & 1)] : 0.f;
    __syncthreads();

    // CTA = 32 vertices x 4 k-slices: warp ks accumulates its quarter of the 350 shape and 36 pose
    // directions for the warp's 32 vertices (each global load is 384 contiguous bytes), partial sums
    // meet in shared memory, then warp ks finishes face t = ks (, ks+4 ...) of the batch tile.
    const int vl = tid & 31, ks = tid >> 5;
    const int v = blockIdx.x * 32 + vl;
    const bool v_ok = v < d.V;
    const int m = 3 * (v_ok ? v : 0);
    float acc[BT][3];
#pragma unroll
    for (int t = 0; t < BT; ++t) { acc[t][0] = 0.f; acc[t][1] = 0.f; acc[t][2] = 0.f; }
    const size_t Mp = d.Mp;
    {   // v_shaped - v_template = shapedirs . beta                                 lbs.py:184,270
        const int per = (d.L + 3) >> 2, l0 = ks * per, l1 = min(d.L, l0 + per);
        const float* sd = d.sdt + m;
#pragma unroll 8
        for (int l = l0; l < l1; ++l) {
            float s0 = __ldg(sd + l * Mp), s1 = __ldg(sd + l * Mp + 1), s2 = __ldg(sd + l * Mp + 2);
#pragma unroll
            for (int t = 0; t < BT; ++t) {
                float be = sB[l * BT + t];
                acc[t][0] = fmaf(s0, be, acc[t][0]);
                acc[t][1] = fmaf(s1, be, acc[t][1]);
                acc[t][2] = fmaf(s2, be, acc[t][2]);
            }
        }
        // + pose_feature . posedirs                                                lbs.py:199-208
        const float* pd = d.pdt + m;
#pragma unroll
        for (int p = ks * 9; p < ks * 9 + 9; ++p) {
            float s0 = __ldg(pd + p * Mp), s1 = __ldg(pd + p * Mp + 1), s2 = __ldg(pd + p * Mp + 2);
#pragma unroll
            for (int t = 0; t < BT; ++t) {
                float f = sP[p * BT + t];
                acc[t][0] = fmaf(s0, f, acc[t][0]);
                acc[t][1] = fmaf(s1, f, acc[t][1]);
                acc[t][2] = fmaf(s2, f, acc[t][2]);
            }
        }
    }
    float* sPart = sE + BT * 2;                     // [4 slices][BT][3][32 lanes]
#pragma unroll
    for (int t = 0; t < BT; ++t)
#pragma unroll
        for (int k = 0; k < 3; ++k) sPart[((ks * BT + t) * 3 + k) * 32 + vl] = acc[t][k];
    __syncthreads();
    if (!v_ok) return;
    // skinning: T = sum_j w_j A_j ; out = T [v_posed;1]                           lbs.py:214-225
    float w[kJ];
#pragma unroll
    for (int j = 0; j < kJ; ++j) w[j] = __ldg(d.wt + (size_t)j * d.V + v);
    const float le0 = d.leye[m], le1 = d.leye[m + 1], le2 = d.leye[m + 2];
    const float re0 = d.reye[m], re1 = d.reye[m + 1], re2 = d.reye[m + 2];
    const float t0 = d.vt[m], t1 = d.vt[m + 1], t2 = d.vt[m + 2];
    for (int t = ks; t < BT; t += 4) {
        if (b0 + t >= B) break;
        float x = t0, y = t1, z = t2;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            x += sPart[((q * BT + t) * 3 + 0) * 32 + vl];
            y += sPart[((q * BT + t) * 3 + 1) * 32 + vl];
            z += sPart[((q * BT + t) * 3 + 2) * 32 + vl];
        }
        float T[12];
#pragma unroll
        for (int e = 0; e < 12; ++e) {
            float a = 0.f;
#pragma unroll
            for (int j = 0; j < kJ; ++j) a = fmaf(w[j], sA[t * 60 + j * 12 + e], a);
            T[e] = a;
        }
        float ox = T[0] * x + T[1] * y + T[2] * z + T[3];
        float oy = T[4] * x + T[5] * y + T[6] * z + T[7];
        float oz = T[8] * x + T[9] * y + T[10] * z + T[11];
        // eyelids are applied after skinning, un-rotated; right (e[:,1]) first   FLAME.py:284-286
        float el = sE[t * 2 + 0], er = sE[t * 2 + 1];
        ox = (ox + re0 * er) + le0 * el;
        oy = (oy + re1 * er) + le1 * el;
        oz = (oz + re2 * er) + le2 * el;
        float* o = verts + ((size_t)(b0 + t) * d.V + v) * 3;
        o[0] = ox; o[1] = oy; o[2] = oz;
    }
}

// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
flame_landmarks_kernel(FlameDev d, const float* __restrict__ verts, const int32_t* __restrict__ dyn_idx, int B,
                       float* __restrict__ lmk_fan, float* __restrict__ lmk_fan3d, float* __restrict__ lmk_mp) {
    const int b = blockIdx.x;
    const int n_fan = d.n_dyn + d.n_static;
    const int total = n_fan + d.n_full + d.n_mp;
    const float* vb = verts + (size_t)b * d.V * 3;
    const int row = dyn_idx[b];
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
        int f; const float* bc; float* out;
        if (i < d.n_dyn) {                                   // 17 dynamic contour + 51 static  FLAME.py:295-296
            f = d.dyn_faces[row * d.n_dyn + i]; bc = d.dyn_bary + ((size_t)row * d.n_dyn + i) * 3;
            out = lmk_fan + ((size_t)b * n_fan + i) * 3;
        } else if (i < n_fan) {
            int k = i - d.n_dyn; f = d.static_faces[k]; bc = d.static_bary + k * 3;
            out = lmk_fan + ((size_t)b * n_fan + i) * 3;
        } else if (i < n_fan + d.n_full) {
            int k = i - n_fan; f = d.full_faces[k]; bc = d.full_bary + k * 3;
            out = lmk_fan3d + ((size_t)b * d.n_full + k) * 3;
        } else {
            int k = i - n_fan - d.n_full; f = d.mp_faces[k]; bc = d.mp_bary + k * 3;
            out = lmk_mp + ((size_t)b * d.n_mp + k) * 3;
        }
        const int32_t* tri = d.faces + (size_t)f * 3;
        const float* p0 = vb + (size_t)tri[0] * 3; const float* p1 = vb + (size_t)tri[1] * 3; const float* p2 = vb + (size_t)tri[2] * 3;
        float w0 = bc[0], w1 = bc[1], w2 = bc[2];
#pragma unroll
        for (int k = 0; k < 3; ++k) out[k] = (p0[k] * w0 + p1[k] * w1) + p2[k] * w2;     // lbs.py:136
    }
}

// =================================================================================================
// Backward: the gradient torch autograd takes through FLAME.forward (FLAME.py:232-315, lbs.py:140-227,
// 274-378) for betas, full_pose and eyelid.  Five launches, no atomics, every reduction in a fixed order:
//   flame_pose_kernel       (the forward's) recomputes the joint transforms A and the pose feature.
//   flame_bwd_posed_kernel  recomputes v_posed = v_template + shapedirs.beta + posedirs.pf.
//   flame_bwd_vert_kernel   per vertex: total upstream g_v (vertices + the landmark gathers of lbs.py:136,
//                           the dynamic contour rows being the forward's dyn_idx), g_vposed = T^T g_v,
//                           and per-CTA partials of g_A = sum_v w_vj g_v [v_posed;1]^T and of the eyelids.
//   flame_bwd_gemv_kernel   g_beta(shape part) = shapedirs^T g_vposed, g_pf = posedirs^T g_vposed.
//   flame_bwd_joint_kernel  per face: sums the partials, backpropagates the kinematic chain
//                           (lbs.py:345-376) and Rodrigues (lbs.py:289-304), adds JS^T g_J (lbs.py:188).
// The contour LUT row (FLAME.py:117-159) is piecewise constant in the pose and contributes no gradient.
struct FlameBwd {
    int32_t* lptr;     // [V+1]  CSR vertex -> fixed landmark corners (static fan, fan3d, mp)
    int32_t* lslot;    //        slot in the concatenated landmark list: fan 0..67, fan3d 68..135, mp 136..
    float* lw;         //        barycentric weight of that corner
};

constexpr int kBwdRows = 4;        // gemv: output rows per CTA
constexpr int kBwdBT = 8;          // gemv / posed: faces per CTA
constexpr int kPart = 62;          // per-CTA partials: g_A (60) + eyelid (2)

__global__ void __launch_bounds__(128)
flame_bwd_posed_kernel(FlameDev d, const float* __restrict__ betas, const float* __restrict__ pf, int B,
                       float* __restrict__ vp /*[B][Mp]*/) {
    // betas + pose feature [(L+36)][kBwdBT] (L <= 350 is checked by the entry point), then the partial sums
    __shared__ __align__(16) float sB[4 * kBwdBT * 32 * 4];
    static_assert((350 + kPF) * kBwdBT <= 4 * kBwdBT * 32 * 4, "flame_bwd_posed_kernel: shared buffer");
    const int b0 = blockIdx.y * kBwdBT, R = d.L + kPF;
    for (int i = threadIdx.x; i < R * kBwdBT; i += 128) {
        int l = i / kBwdBT, t = i % kBwdBT, b = min(b0 + t, B - 1);
        sB[i] = l < d.L ? betas[(size_t)b * d.L + l] : pf[(size_t)b * kPF + (l - d.L)];
    }
    __syncthreads();                                 // every warp reads rows the other warps staged
    // CTA = 32 float4 columns x 4 row slices (as flame_verts_kernel): warp ks sums its quarter of the rows,
    // the partial sums meet in shared memory
    const int lane = threadIdx.x & 31, ks = threadIdx.x >> 5;
    const int m4 = blockIdx.x * 32 + lane;
    const bool ok = m4 * 4 < d.Mp;
    float4 acc[kBwdBT];
#pragma unroll
    for (int t = 0; t < kBwdBT; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int per = (R + 3) >> 2, l0 = ks * per, l1 = min(R, l0 + per);
    if (ok)
        for (int l = l0; l < l1; ++l) {
            const float* row = l < d.L ? d.sdt + (size_t)l * d.Mp : d.pdt + (size_t)(l - d.L) * d.Mp;
            float4 s = __ldg(reinterpret_cast<const float4*>(row) + m4);
#pragma unroll
            for (int t = 0; t < kBwdBT; ++t) smk::fma4_s(acc[t], sB[l * kBwdBT + t], s);
        }
    __syncthreads();                                 // sB is reused for the partial sums
    float4* sPart = reinterpret_cast<float4*>(sB);   // [4 slices][kBwdBT][32 lanes]
#pragma unroll
    for (int t = 0; t < kBwdBT; ++t) sPart[(ks * kBwdBT + t) * 32 + lane] = acc[t];
    __syncthreads();
    if (!ok) return;
    const float4 vt = reinterpret_cast<const float4*>(d.vt)[m4];
    for (int t = ks; t < kBwdBT && b0 + t < B; t += 4) {
        float4 o = vt;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float4 p = sPart[(q * kBwdBT + t) * 32 + lane];
            o.x += p.x; o.y += p.y; o.z += p.z; o.w += p.w;
        }
        reinterpret_cast<float4*>(vp + (size_t)(b0 + t) * d.Mp)[m4] = o;
    }
}

__global__ void __launch_bounds__(128)
flame_bwd_vert_kernel(FlameDev d, FlameBwd bw, const float* __restrict__ A,
                      const float* __restrict__ vp, const int32_t* __restrict__ dyn_idx,
                      const float* __restrict__ g_verts, const float* __restrict__ g_fan,
                      const float* __restrict__ g_fan3d, const float* __restrict__ g_mp, int B,
                      float* __restrict__ gvp /*[B][Mp]*/, double* __restrict__ part /*[B][gridDim.x][62]*/) {
    __shared__ float sA[60];
    __shared__ int32_t sDv[17 * 3];
    __shared__ float sDw[17 * 3];
    __shared__ double sRed[4][kPart];
    const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n_fan = d.n_dyn + d.n_static;
    if (tid < 60) sA[tid] = A[(size_t)b * 60 + tid];
    if (tid < d.n_dyn * 3) {                          // the forward's contour row, expanded to vertex corners
        const int row = dyn_idx[b], i = tid / 3, c = tid % 3;
        const int f = d.dyn_faces[row * d.n_dyn + i];
        sDv[tid] = d.faces[(size_t)f * 3 + c];
        sDw[tid] = d.dyn_bary[((size_t)row * d.n_dyn + i) * 3 + c];
    }
    __syncthreads();
    const int v = blockIdx.x * 128 + tid;
    const bool ok = v < d.V;
    float g[3] = {0.f, 0.f, 0.f}, x[3] = {0.f, 0.f, 0.f}, w[kJ];
    float le[3] = {0.f, 0.f, 0.f}, re[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < kJ; ++j) w[j] = 0.f;
    if (ok) {
        const int m = 3 * v;
        if (g_verts) {
            const float* gv = g_verts + ((size_t)b * d.V + v) * 3;
            g[0] = gv[0]; g[1] = gv[1]; g[2] = gv[2];
        }
        if (g_fan) {                                  // 17 dynamic contour landmarks: lbs.py:136 gathers
            for (int e = 0; e < d.n_dyn * 3; ++e)
                if (sDv[e] == v) {
                    const float* gl = g_fan + ((size_t)b * n_fan + e / 3) * 3;
#pragma unroll
                    for (int k = 0; k < 3; ++k) g[k] = fmaf(sDw[e], gl[k], g[k]);
                }
        }
        for (int e = bw.lptr[v]; e < bw.lptr[v + 1]; ++e) {      // static fan, fan3d, mp landmarks
            const int s = bw.lslot[e];
            const float* gl = s < n_fan ? (g_fan ? g_fan + ((size_t)b * n_fan + s) * 3 : nullptr)
                            : s < n_fan + d.n_full ? (g_fan3d ? g_fan3d + ((size_t)b * d.n_full + s - n_fan) * 3 : nullptr)
                            : (g_mp ? g_mp + ((size_t)b * d.n_mp + s - n_fan - d.n_full) * 3 : nullptr);
            if (!gl) continue;
#pragma unroll
            for (int k = 0; k < 3; ++k) g[k] = fmaf(bw.lw[e], gl[k], g[k]);
        }
        const float* p = vp + (size_t)b * d.Mp + m;
        x[0] = p[0]; x[1] = p[1]; x[2] = p[2];
#pragma unroll
        for (int j = 0; j < kJ; ++j) w[j] = __ldg(d.wt + (size_t)j * d.V + v);
#pragma unroll
        for (int k = 0; k < 3; ++k) { le[k] = d.leye[m + k]; re[k] = d.reye[m + k]; }
        // out = T [v_posed;1], T = sum_j w_j A_j                                    lbs.py:214-225
        float T[12];
#pragma unroll
        for (int e = 0; e < 12; ++e) {
            float a = 0.f;
#pragma unroll
            for (int j = 0; j < kJ; ++j) a = fmaf(w[j], sA[j * 12 + e], a);
            T[e] = a;
        }
        float* o = gvp + (size_t)b * d.Mp + m;
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c] = T[0 * 4 + c] * g[0] + T[1 * 4 + c] * g[1] + T[2 * 4 + c] * g[2];
        if (v == 0)
            for (int q = 3 * d.V; q < d.Mp; ++q) gvp[(size_t)b * d.Mp + q] = 0.f;   // row padding feeds the gemv
    }
    // per-CTA partials: g_A[j][i][c] = sum_v w_j g_i [x;1]_c ; g_eyelid = sum_v (l_eyelid, r_eyelid) . g.
    // In double: the chain backward subtracts g_A_t J^T from g_A_rot, sums over all vertices of similar size.
#pragma unroll 1
    for (int q = 0; q < kPart; ++q) {
        double val;
        if (q < 60) {
            const int j = q / 12, i = (q % 12) / 4, c = q % 4;
            val = (double)w[j] * g[i] * (c < 3 ? x[c] : 1.f);
        } else {
            const float* e = q == 60 ? le : re;
            val = (double)e[0] * g[0] + (double)e[1] * g[1] + (double)e[2] * g[2];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) val += __shfl_xor_sync(0xffffffffu, val, o);
        if (lane == 0) sRed[warp][q] = val;
    }
    __syncthreads();
    if (tid < kPart)
        part[((size_t)b * gridDim.x + blockIdx.x) * kPart + tid] = ((sRed[0][tid] + sRed[1][tid]) + sRed[2][tid]) + sRed[3][tid];
}

// out[b][r] = sum_m row_r[m] * gvp[b][m] for the L shape rows and the 36 posedirs rows (fixed order).
__global__ void __launch_bounds__(256)
flame_bwd_gemv_kernel(FlameDev d, const float* __restrict__ gvp, int B, float* __restrict__ out /*[B][L+36]*/) {
    __shared__ float sRed[8][kBwdRows * kBwdBT];
    const int R = d.L + kPF, r0 = blockIdx.x * kBwdRows, b0 = blockIdx.y * kBwdBT;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float4* rows[kBwdRows];
#pragma unroll
    for (int i = 0; i < kBwdRows; ++i) {
        const int r = min(r0 + i, R - 1);
        rows[i] = reinterpret_cast<const float4*>(r < d.L ? d.sdt + (size_t)r * d.Mp : d.pdt + (size_t)(r - d.L) * d.Mp);
    }
    float acc[kBwdRows][kBwdBT];
#pragma unroll
    for (int i = 0; i < kBwdRows; ++i)
#pragma unroll
        for (int t = 0; t < kBwdBT; ++t) acc[i][t] = 0.f;
    const int M4 = d.Mp >> 2;
    for (int m4 = tid; m4 < M4; m4 += 256) {
        float4 s[kBwdRows];
#pragma unroll
        for (int i = 0; i < kBwdRows; ++i) s[i] = __ldg(rows[i] + m4);
#pragma unroll
        for (int t = 0; t < kBwdBT; ++t) {
            const float4 gv = reinterpret_cast<const float4*>(gvp + (size_t)min(b0 + t, B - 1) * d.Mp)[m4];
#pragma unroll
            for (int i = 0; i < kBwdRows; ++i) {
                float a = acc[i][t];
                a = fmaf(s[i].x, gv.x, a); a = fmaf(s[i].y, gv.y, a); a = fmaf(s[i].z, gv.z, a); a = fmaf(s[i].w, gv.w, a);
                acc[i][t] = a;
            }
        }
    }
#pragma unroll
    for (int i = 0; i < kBwdRows; ++i)
#pragma unroll
        for (int t = 0; t < kBwdBT; ++t) {
            float val = acc[i][t];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) val += __shfl_xor_sync(0xffffffffu, val, o);
            if (lane == 0) sRed[warp][i * kBwdBT + t] = val;
        }
    __syncthreads();
    if (tid < kBwdRows * kBwdBT) {
        const int i = tid / kBwdBT, t = tid % kBwdBT, r = r0 + i, b = b0 + t;
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) s += sRed[k][tid];
        if (r < R && b < B) out[(size_t)b * R + r] = s;
    }
}

// d/dr of rodrigues(r) (lbs.py:289-304) differentiated as written: angle = ||r + 1e-8||, r_hat = r / angle,
// R = I + sin*K(r_hat) + (1-cos)*K*K.  Finite at r = 0 (sin(angle)/angle -> 1).
// Evaluated in double (the angle from the fp32 r + 1e-8f of the forward).
__device__ void rodrigues_bwd(const float* r, const double* gR, float* gr) {
    const double a[3] = {r[0] + 1e-8f, r[1] + 1e-8f, r[2] + 1e-8f};
    double th = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
    double rx = r[0] / th, ry = r[1] / th, rz = r[2] / th;
    double s = sin(th), c = cos(th), omc = 1.0 - c;
    double K[9] = {0.0, -rz, ry, rz, 0.0, -rx, -ry, rx, 0.0};
    double gK[9], gs = 0.0, gomc = 0.0;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double kk = 0.0, gm = 0.0;
            for (int k = 0; k < 3; ++k) {
                kk += K[i * 3 + k] * K[k * 3 + j];
                gm += gR[i * 3 + k] * K[j * 3 + k] + K[k * 3 + i] * gR[k * 3 + j];      // (gM K^T + K^T gM)
            }
            gs += gR[i * 3 + j] * K[i * 3 + j];
            gomc += gR[i * 3 + j] * kk;
            gK[i * 3 + j] = s * gR[i * 3 + j] + omc * gm;
        }
    double gth = gs * c + gomc * s;
    double gh[3] = {gK[7] - gK[5], gK[2] - gK[6], gK[3] - gK[1]};     // K = [[0,-z,y],[z,0,-x],[-y,x,0]]
    double dot = gh[0] * r[0] + gh[1] * r[1] + gh[2] * r[2];
    gth -= dot / (th * th);
    for (int k = 0; k < 3; ++k) gr[k] = (float)(gh[k] / th + gth * a[k] / th);
}

// G = P * [R | t] and its gradient (accumulates into gP, gR and returns gt), in double.
__device__ void affine_mul_d(const double* P, const double* R, const double* t, double* G) {
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) G[i * 4 + j] = P[i * 4 + 0] * R[0 * 3 + j] + P[i * 4 + 1] * R[1 * 3 + j] + P[i * 4 + 2] * R[2 * 3 + j];
        G[i * 4 + 3] = P[i * 4 + 0] * t[0] + P[i * 4 + 1] * t[1] + P[i * 4 + 2] * t[2] + P[i * 4 + 3];
    }
}

__device__ void affine_mul_bwd(const double* P, const double* R, const double* t, const double* gG,
                               double* gP, double* gR, double* gt) {
    for (int i = 0; i < 3; ++i) {
        for (int k = 0; k < 3; ++k) {
            double acc = gG[i * 4 + 3] * t[k];
            for (int c = 0; c < 3; ++c) acc += gG[i * 4 + c] * R[k * 3 + c];
            gP[i * 4 + k] += acc;
        }
        gP[i * 4 + 3] += gG[i * 4 + 3];
    }
    for (int k = 0; k < 3; ++k) {
        for (int c = 0; c < 3; ++c)
            gR[k * 3 + c] += P[0 * 4 + k] * gG[0 * 4 + c] + P[1 * 4 + k] * gG[1 * 4 + c] + P[2 * 4 + k] * gG[2 * 4 + c];
        gt[k] = P[0 * 4 + k] * gG[0 * 4 + 3] + P[1 * 4 + k] * gG[1 * 4 + 3] + P[2 * 4 + k] * gG[2 * 4 + 3];
    }
}

__global__ void __launch_bounds__(128)
flame_bwd_joint_kernel(FlameDev d, const float* __restrict__ betas, const float* __restrict__ full_pose,
                       const double* __restrict__ part, int n_part, const float* __restrict__ gsd, int B,
                       float* __restrict__ g_betas, float* __restrict__ g_pose, float* __restrict__ g_eyelid) {
    __shared__ float sJ[15], sGJ[15];
    __shared__ double sGA[kPart];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int R = d.L + kPF;
    const float* beta = betas + (size_t)b * d.L;
    for (int row = warp; row < 15; row += 4) {                 // J = J0 + JS beta, as in flame_pose_kernel
        const float* js = d.js + (size_t)row * d.L;
        float acc = 0.f;
        for (int l = lane; l < d.L; l += 32) acc = fmaf(js[l], beta[l], acc);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) sJ[row] = d.j0[row] + acc;
    }
    if (tid < kPart) {                                          // partials of flame_bwd_vert_kernel, in CTA order
        double s = 0.0;
        for (int p = 0; p < n_part; ++p) s += part[((size_t)b * n_part + p) * kPart + tid];
        sGA[tid] = s;
    }
    __syncthreads();
    if (tid == 0) {
        // the chain backward runs in double: its terms are sums over all vertices that largely cancel
        double Rm[kJ][9], G[kJ][12], gG[kJ][12], gR[kJ][9], gJ[15];
        for (int j = 0; j < kJ; ++j) {
            float r32[9];
            rodrigues(full_pose + (size_t)b * 15 + j * 3, r32);
            for (int e = 0; e < 9; ++e) Rm[j][e] = r32[e];
        }
        // forward chain (lbs.py:345-363), as flame_pose_kernel
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) G[0][i * 4 + j] = Rm[0][i * 3 + j];
            G[0][i * 4 + 3] = sJ[i];
        }
        double rel[kJ][3];
        for (int k = 0; k < 3; ++k) rel[1][k] = sJ[3 + k] - sJ[k];
        affine_mul_d(G[0], Rm[1], rel[1], G[1]);
        for (int j = 2; j < kJ; ++j) {
            for (int k = 0; k < 3; ++k) rel[j][k] = sJ[3 * j + k] - sJ[3 + k];
            affine_mul_d(G[1], Rm[j], rel[j], G[j]);
        }
        // A = [G_rot | G_t - G_rot J]                                                lbs.py:373-376
        for (int q = 0; q < 15; ++q) gJ[q] = 0.0;
        for (int j = 0; j < kJ; ++j)
            for (int i = 0; i < 3; ++i) {
                const double gt = sGA[j * 12 + i * 4 + 3];
                for (int c = 0; c < 3; ++c) {
                    gG[j][i * 4 + c] = sGA[j * 12 + i * 4 + c] - gt * sJ[3 * j + c];
                    gJ[3 * j + c] -= G[j][i * 4 + c] * gt;
                }
                gG[j][i * 4 + 3] = gt;
            }
        // pose_feature = (R[1:] - I).view(36)                                          lbs.py:197
        for (int e = 0; e < 9; ++e) gR[0][e] = 0.0;
        for (int j = 1; j < kJ; ++j)
            for (int e = 0; e < 9; ++e) gR[j][e] = gsd[(size_t)b * R + d.L + (j - 1) * 9 + e];
        double gt[3];
        for (int j = kJ - 1; j >= 2; --j) {                     // children of joint 1
            affine_mul_bwd(G[1], Rm[j], rel[j], gG[j], gG[1], gR[j], gt);
            for (int k = 0; k < 3; ++k) { gJ[3 * j + k] += gt[k]; gJ[3 + k] -= gt[k]; }
        }
        affine_mul_bwd(G[0], Rm[1], rel[1], gG[1], gG[0], gR[1], gt);
        for (int k = 0; k < 3; ++k) { gJ[3 + k] += gt[k]; gJ[k] -= gt[k]; }
        for (int i = 0; i < 3; ++i) {
            for (int c = 0; c < 3; ++c) gR[0][i * 3 + c] += gG[0][i * 4 + c];
            gJ[i] += gG[0][i * 4 + 3];
        }
        for (int j = 0; j < kJ; ++j) rodrigues_bwd(full_pose + (size_t)b * 15 + j * 3, gR[j], g_pose + (size_t)b * 15 + j * 3);
        for (int q = 0; q < 15; ++q) sGJ[q] = (float)gJ[q];
        if (g_eyelid) { g_eyelid[(size_t)b * 2 + 0] = (float)sGA[60]; g_eyelid[(size_t)b * 2 + 1] = (float)sGA[61]; }
    }
    __syncthreads();
    for (int l = tid; l < d.L; l += 128) {                      // + JS^T g_J  (J = J_regressor v_shaped, lbs.py:188)
        float s = gsd[(size_t)b * R + l];
        for (int q = 0; q < 15; ++q) s = fmaf(d.js[(size_t)q * d.L + l], sGJ[q], s);
        g_betas[(size_t)b * d.L + l] = s;
    }
}

}  // namespace

struct SmkFlame {
    FlameDev d;
    FlameBwd bw;
    smk::DeviceArena arena;
};

extern "C" int smk_flame_create(const SmkFlameDesc* desc, SmkFlame** out) {
    SMK_REQUIRE(desc && out, "smk_flame_create: null argument");
    SMK_REQUIRE(desc->n_joints == kJ, "smk_flame_create: n_joints must be 5 (got %d)", desc->n_joints);
    SMK_REQUIRE(desc->n_verts > 0 && desc->n_betas > 0 && desc->n_faces > 0, "smk_flame_create: bad sizes");
    const int V = desc->n_verts, L = desc->n_betas, M = 3 * V, Mp = (M + 3) & ~3;
    SmkFlame* h = new SmkFlame();
    FlameDev& d = h->d;
    d.V = V; d.F = desc->n_faces; d.L = L; d.Mp = Mp;
    std::vector<float> sdt((size_t)L * Mp, 0.f), pdt((size_t)kPF * Mp, 0.f), vt(Mp, 0.f), wt((size_t)kJ * V), le(Mp, 0.f), re(Mp, 0.f);
    for (int m = 0; m < M; ++m) {
        for (int l = 0; l < L; ++l) sdt[(size_t)l * Mp + m] = desc->shapedirs[(size_t)m * L + l];
        for (int p = 0; p < kPF; ++p) pdt[(size_t)p * Mp + m] = desc->posedirs[(size_t)p * M + m];
        vt[m] = desc->v_template[m]; le[m] = desc->l_eyelid[m]; re[m] = desc->r_eyelid[m];
    }
    for (int v = 0; v < V; ++v) for (int j = 0; j < kJ; ++j) wt[(size_t)j * V + v] = desc->lbs_weights[(size_t)v * kJ + j];
    // pre-contract the joint regressor with the shape basis (double accumulation on the host)
    std::vector<float> js((size_t)15 * L), j0(15);
    {
        std::vector<double> acc((size_t)15 * L, 0.0), a0(15, 0.0);
        for (int j = 0; j < kJ; ++j)
            for (int v = 0; v < V; ++v) {
                double r = desc->J_regressor[(size_t)j * V + v];
                if (r == 0.0) continue;
                for (int k = 0; k < 3; ++k) {
                    a0[j * 3 + k] += r * desc->v_template[v * 3 + k];
                    const float* s = desc->shapedirs + ((size_t)v * 3 + k) * L;
                    double* a = &acc[(size_t)(j * 3 + k) * L];
                    for (int l = 0; l < L; ++l) a[l] += r * s[l];
                }
            }
        for (size_t i = 0; i < acc.size(); ++i) js[i] = (float)acc[i];
        for (int i = 0; i < 15; ++i) j0[i] = (float)a0[i];
    }
    cudaError_t e = cudaSuccess;
    auto up = [&](auto& vec, auto** dst) { if (e == cudaSuccess) e = h->arena.upload(vec, dst); };
    up(sdt, &d.sdt); up(pdt, &d.pdt); up(vt, &d.vt); up(wt, &d.wt); up(le, &d.leye); up(re, &d.reye); up(js, &d.js); up(j0, &d.j0);
    auto upi = [&](const int32_t* p, size_t n, int32_t** dst) { if (e == cudaSuccess) e = h->arena.upload(p, n, dst); };
    auto upf = [&](const float* p, size_t n, float** dst) { if (e == cudaSuccess) e = h->arena.upload(p, n, dst); };
    upi(desc->faces, (size_t)d.F * 3, &d.faces);
    d.n_static = desc->n_static; d.n_dyn_rows = desc->n_dyn_rows; d.n_dyn = desc->n_dyn; d.n_full = desc->n_full; d.n_mp = desc->n_mp;
    upi(desc->static_faces, d.n_static, &d.static_faces); upf(desc->static_bary, (size_t)d.n_static * 3, &d.static_bary);
    upi(desc->dyn_faces, (size_t)d.n_dyn_rows * d.n_dyn, &d.dyn_faces); upf(desc->dyn_bary, (size_t)d.n_dyn_rows * d.n_dyn * 3, &d.dyn_bary);
    upi(desc->full_faces, d.n_full, &d.full_faces); upf(desc->full_bary, (size_t)d.n_full * 3, &d.full_bary);
    upi(desc->mp_faces, d.n_mp, &d.mp_faces); upf(desc->mp_bary, (size_t)d.n_mp * 3, &d.mp_bary);
    {   // backward: CSR vertex -> corners of the fixed landmarks (static fan, fan3d, mp), in slot order
        std::vector<int32_t> cnt(V + 1, 0), lslot;
        std::vector<float> lw;
        auto each = [&](auto fn) {
            const int n_fan = d.n_dyn + d.n_static;
            for (int k = 0; k < d.n_static; ++k) for (int c = 0; c < 3; ++c) fn(desc->faces[desc->static_faces[k] * 3 + c], d.n_dyn + k, desc->static_bary[k * 3 + c]);
            for (int k = 0; k < d.n_full; ++k) for (int c = 0; c < 3; ++c) fn(desc->faces[desc->full_faces[k] * 3 + c], n_fan + k, desc->full_bary[k * 3 + c]);
            for (int k = 0; k < d.n_mp; ++k) for (int c = 0; c < 3; ++c) fn(desc->faces[desc->mp_faces[k] * 3 + c], n_fan + d.n_full + k, desc->mp_bary[k * 3 + c]);
        };
        each([&](int v, int, float) { cnt[v + 1]++; });
        for (int v = 0; v < V; ++v) cnt[v + 1] += cnt[v];
        std::vector<int32_t> fill(cnt.begin(), cnt.end() - 1);
        lslot.resize(cnt[V]); lw.resize(cnt[V]);
        each([&](int v, int s, float w) { lslot[fill[v]] = s; lw[fill[v]++] = w; });
        if (lslot.empty()) { lslot.push_back(0); lw.push_back(0.f); }
        up(cnt, &h->bw.lptr); up(lslot, &h->bw.lslot); up(lw, &h->bw.lw);
    }
    if (e != cudaSuccess) { smk::set_error("smk_flame_create: upload failed: %s", cudaGetErrorString(e)); delete h; return (int)e; }
    *out = h;
    return 0;
}

extern "C" void smk_flame_destroy(SmkFlame* h) { delete h; }

extern "C" size_t smk_flame_workspace_bytes(const SmkFlame*, int B) {
    return smk::ws_round((size_t)B * 60 * 4) + smk::ws_round((size_t)B * kPF * 4) + smk::ws_round((size_t)B * 4);
}

template <int BT>
static int launch_verts(const FlameDev& d, const float* betas, const float* eyelid, const float* A, const float* pf,
                        int B, float* verts, cudaStream_t st) {
    size_t smem = ((size_t)d.L * BT + kPF * BT + BT * 60 + BT * 2 + 4 * BT * 3 * 32) * sizeof(float);
    if (smem > 48 * 1024)
        SMK_CHECK_CUDA(cudaFuncSetAttribute(flame_verts_kernel<BT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(smk::cdiv(d.V, 32), smk::cdiv(B, BT));          // 32 vertices x 4 k-slices per CTA
    SMK_TAG("flame_verts", 4.0 * ((double)(d.L + kPF) * d.Mp + 6.0 * d.Mp + 5.0 * d.V + (double)B * (d.L + 3.0 * d.V + 98)),
            2.0 * B * (3.0 * d.V * (d.L + kPF) + (double)d.V * (60 + 12 + 6)), st);
    SMK_LAUNCH((flame_verts_kernel<BT>), dim3(grid), dim3(128), smem, st, d, betas, eyelid, A, pf, B, verts);
    SMK_CHECK_LAUNCH();
    return 0;
}

extern "C" int smk_flame_forward(const SmkFlame* h, const float* betas, const float* full_pose, const float* eyelid,
                                 int B, float* verts, float* lmk_fan, float* lmk_fan3d, float* lmk_mp,
                                 float* joints, int32_t* dyn_idx, void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;                      // empty batch: nothing to do (pointers may be null)
    SMK_REQUIRE(h && betas && full_pose && verts && lmk_fan && lmk_fan3d && lmk_mp, "smk_flame_forward: null argument");
    SMK_REQUIRE(B > 0, "smk_flame_forward: negative batch");
    SMK_REQUIRE(ws && ws_bytes >= smk_flame_workspace_bytes(h, B), "smk_flame_forward: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    smk::Workspace w(ws, ws_bytes);
    float* A = w.take<float>((size_t)B * 60);
    float* pf = w.take<float>((size_t)B * kPF);
    int32_t* dyn = w.take<int32_t>(B);
    const FlameDev& d = h->d;
    SMK_TAG("flame_pose", 4.0 * (15.0 * d.L + (double)B * (d.L + 15 + 60 + kPF + 16)), 2.0 * B * 15.0 * d.L, st);
    SMK_LAUNCH(flame_pose_kernel, dim3(B), dim3(128), 0, st, d, betas, full_pose, B, A, pf, joints, dyn);
    SMK_CHECK_LAUNCH();
    int rc;
    constexpr int kBt8From = 96;               // batch size from which flame_verts keeps 8 (instead of 4) faces per thread
    if (B >= kBt8From) rc = launch_verts<8>(d, betas, eyelid, A, pf, B, verts, st);
    else if (B >= 8) rc = launch_verts<4>(d, betas, eyelid, A, pf, B, verts, st);
    else if (B >= 2) rc = launch_verts<2>(d, betas, eyelid, A, pf, B, verts, st);
    else rc = launch_verts<1>(d, betas, eyelid, A, pf, B, verts, st);
    if (rc) return rc;
    SMK_TAG("flame_landmarks", 4.0 * B * 241.0 * (9 + 3 + 3 + 4), 2.0 * B * 241 * 9, st);
    SMK_LAUNCH(flame_landmarks_kernel, dim3(B), dim3(256), 0, st, d, verts, dyn, B, lmk_fan, lmk_fan3d, lmk_mp);
    SMK_CHECK_LAUNCH();
    if (dyn_idx) SMK_CHECK_CUDA(cudaMemcpyAsync(dyn_idx, dyn, (size_t)B * 4, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// ---- backward ------------------------------------------------------------------------------------
static int flame_bwd_parts(const FlameDev& d) { return smk::cdiv(d.V, 128); }

extern "C" size_t smk_flame_backward_workspace_bytes(const SmkFlame* h, int B) {
    if (!h || B <= 0) return 0;
    const FlameDev& d = h->d;
    return smk::ws_round((size_t)B * 60 * 4) + smk::ws_round((size_t)B * kPF * 4) + smk::ws_round((size_t)B * d.Mp * 4) * 2 +
           smk::ws_round((size_t)B * flame_bwd_parts(d) * kPart * 8) + smk::ws_round((size_t)B * (d.L + kPF) * 4);
}

extern "C" int smk_flame_backward(const SmkFlame* h, const float* betas, const float* full_pose, const float* eyelid,
                                  int B, const int32_t* dyn_idx, const float* g_verts, const float* g_lmk_fan,
                                  const float* g_lmk_fan3d, const float* g_lmk_mp, float* g_betas, float* g_full_pose,
                                  float* g_eyelid, void* ws, size_t ws_bytes, void* stream) {
    (void)eyelid;                              // eyelids enter linearly: their value does not reach any gradient
    if (B == 0) return 0;
    SMK_REQUIRE(h && betas && full_pose && dyn_idx && g_betas && g_full_pose, "smk_flame_backward: null argument");
    SMK_REQUIRE(B > 0, "smk_flame_backward: negative batch");
    SMK_REQUIRE(ws && ws_bytes >= smk_flame_backward_workspace_bytes(h, B), "smk_flame_backward: workspace too small");
    const FlameDev& d = h->d;
    SMK_REQUIRE(d.L <= 350 && d.n_dyn <= 17, "smk_flame_backward: n_betas <= 350 and 17 contour landmarks supported (got %d, %d)", d.L, d.n_dyn);
    cudaStream_t st = (cudaStream_t)stream;
    smk::Workspace w(ws, ws_bytes);
    float* A = w.take<float>((size_t)B * 60);
    float* pf = w.take<float>((size_t)B * kPF);
    float* vp = w.take<float>((size_t)B * d.Mp);
    float* gvp = w.take<float>((size_t)B * d.Mp);
    const int np = flame_bwd_parts(d), R = d.L + kPF;
    double* part = w.take<double>((size_t)B * np * kPart);
    float* gsd = w.take<float>((size_t)B * R);
    SMK_TAG("flame_bwd_pose", 4.0 * (15.0 * d.L + (double)B * (d.L + 15 + 60 + kPF)), 2.0 * B * 15.0 * d.L, st);
    SMK_LAUNCH(flame_pose_kernel, dim3(B), dim3(128), 0, st, d, betas, full_pose, B, A, pf, (float*)nullptr, (int32_t*)nullptr);
    SMK_CHECK_LAUNCH();
    SMK_TAG("flame_bwd_posed", 4.0 * ((double)R * d.Mp * smk::cdiv(B, kBwdBT) + (double)B * (R + d.Mp)), 2.0 * B * (double)R * d.Mp, st);
    SMK_LAUNCH(flame_bwd_posed_kernel, dim3(smk::cdiv(d.Mp / 4, 32), smk::cdiv(B, kBwdBT)), dim3(128), 0, st, d, betas, pf, B, vp);
    SMK_CHECK_LAUNCH();
    SMK_TAG("flame_bwd_vert", 4.0 * ((double)B * (d.Mp * 2.0 + (g_verts ? 3.0 * d.V : 0.0) + 2.0 * np * kPart) + 14.0 * d.V),
            2.0 * B * (double)d.V * (60 + 9 + 60 + 6), st);
    SMK_LAUNCH(flame_bwd_vert_kernel, dim3(np, B), dim3(128), 0, st, d, h->bw, A, vp, dyn_idx, g_verts, g_lmk_fan,
               g_lmk_fan3d, g_lmk_mp, B, gvp, part);
    SMK_CHECK_LAUNCH();
    SMK_TAG("flame_bwd_gemv", 4.0 * ((double)R * d.Mp * smk::cdiv(B, kBwdBT) + (double)B * d.Mp * smk::cdiv(R, kBwdRows) + (double)B * R),
            2.0 * B * (double)R * d.Mp, st);
    SMK_LAUNCH(flame_bwd_gemv_kernel, dim3(smk::cdiv(R, kBwdRows), smk::cdiv(B, kBwdBT)), dim3(256), 0, st, d, gvp, B, gsd);
    SMK_CHECK_LAUNCH();
    SMK_TAG("flame_bwd_joint", 4.0 * ((double)B * (2.0 * np * kPart + 2.0 * d.L + R + 17) + 16.0 * d.L), 2.0 * B * 30.0 * d.L, st);
    SMK_LAUNCH(flame_bwd_joint_kernel, dim3(B), dim3(128), 0, st, d, betas, full_pose, part, np, gsd, B, g_betas, g_full_pose, g_eyelid);
    SMK_CHECK_LAUNCH();
    return 0;
}
