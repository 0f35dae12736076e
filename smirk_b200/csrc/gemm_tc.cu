// TF32 tensor-core implicit-GEMM convolution for sm_90a (Hopper wgmma):  C[M,N] = epi( A[M,K] * W[N,K]^T ).
//
// This is the tensor-core path of the generator's 3x3 convolutions / transposed convolutions and of
// the encoder's 1x1 convolutions (precision = 1; the 3xTF32 instantiations at precision 3).  The reference executes
// these layers as cuDNN TF32 implicit GEMMs (src/smirk_generator.py:56-76,147-178; torch default cudnn.allow_tf32=True);
// here they are one hand-written kernel:
//
//   * A (activations, NHWC fp32) is fetched tile-by-tile by TMA: `cp.async.bulk.tensor.2d` for 1x1
//     convs / plain GEMMs, `cp.async.bulk.tensor.4d...im2col` for 3x3 convs — the hardware walks 128
//     consecutive output pixels (crossing rows and images), applies the filter-tap offset and zero
//     fills the padding halo, writing a 128 x 32-channel (128-byte rows) SWIZZLE_128B tile into
//     shared memory.  No im2col matrix is ever materialised.
//   * W ([N][K], K-major, K ordered (tap, channel)) comes in through a 2-D TMA box of BN x 32.
//   * Two consumer warpgroups each own 64 rows of the 128-row tile and issue
//     `wgmma.mma_async.m64nBNk8.f32.tf32.tf32` from shared-memory descriptors (4 per 128-byte k-block); the fp32
//     accumulators live in registers (BN / 2 per thread).
//   * A STAGES-deep mbarrier ring decouples the TMA producer warp from the consumers; a consumer releases a stage
//     as soon as the wgmma group that read it has retired (one group stays in flight).  The epilogue — folded
//     BatchNorm scale/bias, optional residual and ReLU, NHWC stores plain, into a channel slice of a concat buffer,
//     into the interior of a reflection-padded buffer, or pixel-shuffled (ConvTranspose2d k2 s2) — runs in the same
//     warps, straight from the accumulator registers through a per-warp staging slab.
//
// Threads (288): warps 0..7 = consumers (warpgroups 0 and 1), warp 8 = TMA producer.
#include "gemm_tc.cuh"
#include "tc_ptx.cuh"

namespace smk {
namespace {

constexpr int BM = 128;
constexpr int BKB = 128;                  // bytes of K per k-block = one SWIZZLE_128B row = 32 fp32
constexpr int BK = 32;
constexpr int MMA_K = 8;                  // tf32
constexpr int A_STAGE_BYTES = BM * BKB;   // 16 KiB
constexpr int CONSUMER_WARPS = 8;
constexpr int NUM_THREADS = CONSUMER_WARPS * 32 + 32;
constexpr int SLAB_BYTES = CONSUMER_WARPS * 2048;     // epilogue staging: 16 rows x 128 B per consumer warp
constexpr int BAR_BYTES = 256;
constexpr int HEAD_PAR_BYTES = 1088;                  // store 3: [32][8] per-channel constants + 4 head biases

using namespace ptx;                      // PTX wrappers shared by the tensor-core kernels (tc_ptx.cuh)

struct TcArgs {
    int M, N, nkb;                 // nkb = number of 32-wide k-blocks
    int tiles_n, n_tiles;          // column tiles per row of tiles, total tiles (tile t -> row tile t / tiles_n)
    int mode;                      // 0 = 2-D tiled A; 1 = im2col A
    int H, W;                      // output spatial dims (im2col tile origin decode; shuffle / padded stores)
    int cpb;                       // k-blocks per filter tap (Cin / 32) for im2col
    int lc;                        // im2col lower corner (-1: zero padding 1; 0: input already reflection-padded)
    // Two problems of identical shape may share one launch (the encoder's two "large" backbones run the same layer
    // list on different weights and activations): tiles [0, n_tiles_g) belong to problem 0, [n_tiles_g, 2 n_tiles_g) to
    // problem 1, each with its own tensor maps (TcMaps) and epilogue pointers.  Twice the work per launch for kernels
    // that sit on the launch/latency floor.
    int n_tiles_g;                 // tiles per problem (= n_tiles when there is only one)
    const float* scale[2]; const float* bias[2];
    const float* res[2]; int ld_res; int res_pad;   // residual (optionally read from the interior of a padded buffer)
    int relu;
    float* out[2]; int ld_out;
    int store;                     // 0 plain, 1 pixel-shuffle (N = 4*Cout), 2 interior of a (H+2)x(W+2) padded buffer,
                                   // 3 fused head: out[b, co, h, w] = sigmoid(head_b[co] + sum_n act[m, n] * head_w[n][co]) (NCHW, N <= 32)
    int round_out;                 // 1: round the stored activations to TF32 (round-to-nearest) for the next tensor-core layer
    const float* head_w; const float* head_b; int head_c;      // store 3: 1x1 head weights [N][head_c], bias [head_c], head_c <= 4
    const float* mask; int ld_mask;    // zero outputs whose mask[m, n] <= 0 (single problem, store 0)
    float* out2; int ld_out2;          // second store of the activations, compact at pixel m (single problem, store 0 / 2 / 3)
    int out2_rows;                     // out2 takes the pixels m < out2_rows
    const float* prelu;                // PReLU slope per column (AFF instantiations; store 0)
    const float* scale2; const float* bias2; int round_out2;   // out2 = scale2 * v + bias2 of the unrounded v (AFF)
};

struct TcMaps { CUtensorMap a[2], b[2], blo[2]; };       // per problem: activations, weights (TF32 heads), weight tails (3xTF32)

template <int BN, int STAGES, int MINB, bool PERSIST, int X3, bool EXTRA, bool AFF = false>
__global__ void __launch_bounds__(NUM_THREADS, MINB)
gemm_tc_kernel(const __grid_constant__ TcMaps mp, const TcArgs a) {
    // Output tiles (128 rows x BN columns) are strided over the grid.
    //   PERSIST = true : grid = resident CTAs; the smem ring runs across tile boundaries, so the TMA loads of tile i+1
    //                    are in flight while the consumers run the epilogue of tile i.
    //   PERSIST = false: grid = tiles, one tile per CTA, and each consumer warp's staging slab aliases the A rows of ring
    //                    stage 0 that only its own warpgroup reads (and has finished reading when the epilogue starts):
    //                    a smaller footprint, so more CTAs of this kernel and of the concurrent pipeline's other kernels
    //                    share an SM, which is what the shallow-K streaming 1x1 layers want.
    //   X3 = 2         : error-compensated "3xTF32" arithmetic (fp32-equivalent results on the tensor cores).  Every fp32
    //                    operand is split into a TF32 head and a TF32 tail, a = a_hi + a_lo, and three products are
    //                    accumulated: a_hi*w_hi + a_lo*w_hi + a_hi*w_lo (the dropped a_lo*w_lo term is ~2^-22 relative).
    //                    Weights are split on the host (TcMaps::blo maps the tails).  The activation tile is split in
    //                    registers by the consumers (A fragments of the register form of wgmma), so shared memory holds
    //                    only the plain kernel's tiles plus the weight tails.
    //   X3 = 3         : 3xTF32 for deep K (the generator's convolutions, K up to 4608).  The tensor core's accumulator
    //                    truncates at every wgmma update, and with 3 K / 8 updates into one running sum those losses add
    //                    up to ~2^-22 K / 8 of the output scale (1e-4 at K = 4608, TF32's order over a network).  Here each
    //                    k-block's 12 updates go into a fresh register tile that is then added to the running sum by an
    //                    fp32 (round-to-nearest) add: the truncation only ever sees one k-block's partial sum.
    //   EXTRA = true     : the epilogue also applies `mask` and writes `out2` (backward / grad-mode forward); the forward-only
    //                    instantiations are compiled without them.
    //   AFF = true       : (with EXTRA) also the per-column PReLU and the second store's own affine (MICA's residual blocks).
    static_assert(!X3 || !PERSIST, "3xTF32 runs single-tile CTAs");
    constexpr int B_STAGE_BYTES = BN * BKB;
    constexpr int HALF_STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
    constexpr int STAGE_BYTES = X3 ? HALF_STAGE_BYTES + B_STAGE_BYTES : HALF_STAGE_BYTES;         // [A][B] (+ [B tails])
    constexpr int BLO_OFF = HALF_STAGE_BYTES;                                                       // weight tails within a stage
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for SWIZZLE_128B; offset arithmetic keeps the shared address space visible to the
    // compiler (LDS/STS for the staging slab instead of generic LD/ST).
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* slabs = PERSIST ? smem + STAGES * STAGE_BYTES : smem;      // 8 x 2 KiB epilogue staging, one per consumer warp
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + (PERSIST ? SLAB_BYTES : 0));
    uint64_t* empty = full + STAGES;
    float* hpar = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(full) + BAR_BYTES);   // store 3 constants

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == CONSUMER_WARPS && lane == 0) {
        const int g0 = (!PERSIST && (int)blockIdx.x >= a.n_tiles_g) ? 1 : 0;
        prefetch_tensormap(&mp.a[g0]);
        prefetch_tensormap(&mp.b[g0]);
        if (X3) prefetch_tensormap(&mp.blo[g0]);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], CONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == CONSUMER_WARPS) {
        if (lane == 0) {
            // ===== TMA producer =====
            int it = 0;
            for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
                const int g = t >= a.n_tiles_g ? 1 : 0, tt = t - g * a.n_tiles_g;
                const CUtensorMap* tmA = &mp.a[g]; const CUtensorMap* tmB = &mp.b[g]; const CUtensorMap* tmBlo = &mp.blo[g];
                const int tm = tt / a.tiles_n, tn = tt - tm * a.tiles_n;
                const int m0 = tm * BM, n0 = tn * BN;
                int q0 = 0, p0 = 0, img = 0;
                if (a.mode == 1) { int hw = a.H * a.W; img = m0 / hw; int r = m0 - img * hw; p0 = r / a.W; q0 = r - p0 * a.W; }
                for (int kb = 0; kb < a.nkb; ++kb, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(&empty[s], ((uint32_t)(it / STAGES) & 1u) ^ 1u);
                    uint8_t* sa = smem + s * STAGE_BYTES;
                    uint8_t* sb = sa + A_STAGE_BYTES;
                    mbar_expect_tx(&full[s], (uint32_t)(HALF_STAGE_BYTES + (X3 ? B_STAGE_BYTES : 0)));
                    if (X3) tma_load_2d(tmBlo, sa + BLO_OFF, &full[s], kb * BK, n0);
                    if (a.mode == 0) {
                        tma_load_2d(tmA, sa, &full[s], kb * BK, m0);
                    } else {
                        int tap = kb / a.cpb, ch = kb - tap * a.cpb;
                        int r = tap / 3, sx = tap - r * 3;
                        tma_load_im2col(tmA, sa, &full[s], ch * BK, q0 + a.lc, p0 + a.lc, img, (uint16_t)sx, (uint16_t)r);
                    }
                    tma_load_2d(tmB, sb, &full[s], kb * BK, n0);
                }
            }
        }
        return;
    }

    // ===== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64); warp wq of it rows [64 wg + 16 wq, +16) =====
    const int wg = warp >> 2, wq = warp & 3;
    if (a.store == 3) {                                    // head constants of channel `lane` (read-only, shared by all warps)
        if (warp == 0) {
            hpar[lane * 8 + 0] = __ldg(a.scale[0] + lane); hpar[lane * 8 + 1] = __ldg(a.bias[0] + lane);
#pragma unroll
            for (int co = 0; co < 4; ++co) hpar[lane * 8 + 2 + co] = co < a.head_c ? __ldg(a.head_w + (size_t)lane * a.head_c + co) : 0.f;
            if (lane < 4) hpar[256 + lane] = lane < a.head_c ? __ldg(a.head_b + lane) : 0.f;
        }
        named_barrier(1, CONSUMER_WARPS * 32);
    }
    uint8_t* slab = slabs + warp * 2048;
    const int sub = lane >> 3, jj = lane & 7;              // phase-2 role: row-in-group, 16-byte chunk
    int it = 0;
    for (int t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
        const int g = t >= a.n_tiles_g ? 1 : 0, tt = t - g * a.n_tiles_g;
        const int tm = tt / a.tiles_n, tn = tt - tm * a.tiles_n;
        const int m0 = tm * BM, n0 = tn * BN;
        float d[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < a.nkb; ++kb, ++it) {
            const int s = it % STAGES;
            mbar_wait(&full[s], (uint32_t)(it / STAGES) & 1u);
            uint8_t* st = smem + s * STAGE_BYTES;
            const uint32_t sa = smem_u32(st) + (uint32_t)(wg * 64 * BKB);
            const uint32_t sb = smem_u32(st) + A_STAGE_BYTES;
            if constexpr (X3 == 2) {
                uint32_t hi[BK / MMA_K][4], lo[BK / MMA_K][4];
#pragma unroll
                for (int k = 0; k < BK / MMA_K; ++k) {
                    float v[4];
                    load_a_frag(st, wg * 64, k * MMA_K, wq, lane, v);
                    split_frag(v, hi[k], lo[k]);
                }
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / MMA_K; ++k) {
                    const uint64_t db = make_smem_desc(sb + k * MMA_K * 4);
                    const uint64_t dbl = make_smem_desc(smem_u32(st) + BLO_OFF + k * MMA_K * 4);
                    Wgmma<BN>::rs(d, hi[k], db, 1u);                 // a_hi * w_hi
                    Wgmma<BN>::rs(d, lo[k], db, 1u);                 // a_lo * w_hi
                    Wgmma<BN>::rs(d, hi[k], dbl, 1u);                // a_hi * w_lo
                }
                wgmma_commit();
                wgmma_wait<0>();
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);
            } else if constexpr (X3 == 3) {
                // as X3 = 2, into a zeroed tile dk, then d += dk in fp32
                float dk[BN / 2];
                uint32_t hi[BK / MMA_K][4], lo[BK / MMA_K][4];
#pragma unroll
                for (int k = 0; k < BK / MMA_K; ++k) {
                    float v[4];
                    load_a_frag(st, wg * 64, k * MMA_K, wq, lane, v);
                    split_frag(v, hi[k], lo[k]);
                }
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) dk[i] = 0.f;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / MMA_K; ++k) {
                    const uint64_t db = make_smem_desc(sb + k * MMA_K * 4);
                    const uint64_t dbl = make_smem_desc(smem_u32(st) + BLO_OFF + k * MMA_K * 4);
                    Wgmma<BN>::rs(dk, hi[k], db, 1u);
                    Wgmma<BN>::rs(dk, lo[k], db, 1u);
                    Wgmma<BN>::rs(dk, hi[k], dbl, 1u);
                }
                wgmma_commit();
                wgmma_wait<0>();
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) d[i] += dk[i];
            } else {
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / MMA_K; ++k)
                    Wgmma<BN>::ss(d, make_smem_desc(sa + k * MMA_K * 4), make_smem_desc(sb + k * MMA_K * 4), 1u);
                wgmma_commit();
                wgmma_wait<1>();                               // the previous k-block's group has retired: release its stage
                __syncwarp();
                if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
                prev = s;
            }
        }
        if constexpr (X3 == 0) {
            wgmma_wait<0>();
            __syncwarp();
            if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        }

        // ===== epilogue: per 32-column chunk, (1) accumulators -> this warp's slab, (2) 8 lanes per row, 4 rows per
        // instruction: scale/bias (+residual) (+ReLU) (+TF32 rounding) and whole-128-byte-line stores =====
        const float* __restrict__ g_scale = a.scale[g]; const float* __restrict__ g_bias = a.bias[g];
        const float* __restrict__ g_res = a.res[g]; float* __restrict__ g_out = a.out[g];
        const int row0 = m0 + wg * 64 + wq * 16;           // first tile row of this warp
        int opix[4], rpix[4];                              // destination / residual pixel of my 4 phase-2 rows (-1: past M)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int m = row0 + 4 * i + sub;
            int o = -1, r = -1;
            if (m < a.M) {
                o = r = m;
                if (a.store != 0 || a.res_pad) {
                    const int hw = a.H * a.W, b = m / hw, rem = m - b * hw, h = rem / a.W, w = rem - h * a.W;
                    const int padded = (b * (a.H + 2) + h + 1) * (a.W + 2) + w + 1;
                    if (a.store == 2) o = padded;
                    else if (a.store == 1) o = (b * (2 * a.H) + 2 * h) * (2 * a.W) + 2 * w;
                    if (a.res_pad) r = padded;
                }
            }
            opix[i] = o; rpix[i] = r;
        }
#pragma unroll
        for (int c0 = 0; c0 < BN; c0 += 32) {
            const int n = n0 + c0;
            if (n >= a.N) break;                           // warp-uniform
            stage32<BN>(slab, d, c0, lane);
            __syncwarp();
            if (a.store == 3) {
                // Fused 1x1 head + sigmoid (smirk_generator.py:77-78 -> :86), N == BN == 32: lane r < 16 takes slab row r = one
                // pixel with all 32 accumulators; per-channel constants by broadcast LDS; the activation tensor is never written.
                const int m = row0 + lane;
                if (lane < 16 && m < a.M) {
                    float a0 = hpar[256], a1 = hpar[257], a2 = hpar[258], a3 = hpar[259];       // head bias
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float4 x4 = slab_chunk(slab, lane, j);
                        float xs[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int nn = 4 * j + e;
                            const float4 p0 = *reinterpret_cast<const float4*>(hpar + nn * 8);
                            const float2 p1 = *reinterpret_cast<const float2*>(hpar + nn * 8 + 4);
                            float x = fmaf(xs[e], p0.x, p0.y);
                            if (a.relu) x = fmaxf(x, 0.f);
                            xs[e] = x;
                            a0 = fmaf(x, p0.z, a0); a1 = fmaf(x, p0.w, a1); a2 = fmaf(x, p1.x, a2); a3 = fmaf(x, p1.y, a3);
                        }
                        if (EXTRA && a.out2 && m < a.out2_rows) *reinterpret_cast<float4*>(a.out2 + (size_t)m * a.ld_out2 + 4 * j) = make_float4(xs[0], xs[1], xs[2], xs[3]);
                    }
                    const int hw_px = a.H * a.W, b = m / hw_px, rem = m - b * hw_px;
                    float* dst = g_out + (size_t)b * a.head_c * hw_px + rem;
                    dst[0] = 1.f / (1.f + __expf(-a0));
                    if (a.head_c > 1) dst[hw_px] = 1.f / (1.f + __expf(-a1));
                    if (a.head_c > 2) dst[2 * (size_t)hw_px] = 1.f / (1.f + __expf(-a2));
                    if (a.head_c > 3) dst[3 * (size_t)hw_px] = 1.f / (1.f + __expf(-a3));
                }
                __syncwarp();
                continue;
            }
            const int nc = n + jj * 4;                     // my 4 columns
            if (nc < a.N) {
                const float4 sc = __ldg(reinterpret_cast<const float4*>(g_scale + nc));
                const float4 bi = __ldg(reinterpret_cast<const float4*>(g_bias + nc));
                int col = nc, pix_off = 0;
                if (a.store == 1) {                        // ConvTranspose2d k2 s2: n = (dy*2+dx)*Cout + co
                    const int cout = a.N >> 2, q = nc / cout;
                    col = nc - q * cout; pix_off = (q >> 1) * (2 * a.W) + (q & 1);
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if (opix[i] < 0) continue;
                    const float4 x = slab_chunk(slab, 4 * i + sub, jj);
                    float4 o;
                    o.x = fmaf(x.x, sc.x, bi.x); o.y = fmaf(x.y, sc.y, bi.y); o.z = fmaf(x.z, sc.z, bi.z); o.w = fmaf(x.w, sc.w, bi.w);
                    if (g_res) {
                        const float4 r4 = __ldg(reinterpret_cast<const float4*>(g_res + (size_t)rpix[i] * a.ld_res + nc));
                        o.x += r4.x; o.y += r4.y; o.z += r4.z; o.w += r4.w;
                    }
                    if (a.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
                    if constexpr (AFF) {
                        if (a.prelu) {
                            const float4 w4 = __ldg(reinterpret_cast<const float4*>(a.prelu + nc));
                            o.x = o.x < 0.f ? o.x * w4.x : o.x; o.y = o.y < 0.f ? o.y * w4.y : o.y;
                            o.z = o.z < 0.f ? o.z * w4.z : o.z; o.w = o.w < 0.f ? o.w * w4.w : o.w;
                        }
                    }
                    const size_t mc = (size_t)(row0 + 4 * i + sub);            // compact pixel (mask, second store)
                    if (EXTRA && a.mask) {
                        const float4 k4 = __ldg(reinterpret_cast<const float4*>(a.mask + mc * a.ld_mask + nc));
                        o.x = k4.x > 0.f ? o.x : 0.f; o.y = k4.y > 0.f ? o.y : 0.f; o.z = k4.z > 0.f ? o.z : 0.f; o.w = k4.w > 0.f ? o.w : 0.f;
                    }
                    float4 o2 = o;
                    if constexpr (AFF) {
                        if (a.scale2) {
                            const float4 s2 = __ldg(reinterpret_cast<const float4*>(a.scale2 + nc));
                            const float4 b2 = __ldg(reinterpret_cast<const float4*>(a.bias2 + nc));
                            o2.x = fmaf(o.x, s2.x, b2.x); o2.y = fmaf(o.y, s2.y, b2.y); o2.z = fmaf(o.z, s2.z, b2.z); o2.w = fmaf(o.w, s2.w, b2.w);
                            if (a.round_out2) { o2.x = smk::round_tf32(o2.x); o2.y = smk::round_tf32(o2.y); o2.z = smk::round_tf32(o2.z); o2.w = smk::round_tf32(o2.w); }
                        }
                    }
                    if (a.round_out) { o.x = smk::round_tf32(o.x); o.y = smk::round_tf32(o.y); o.z = smk::round_tf32(o.z); o.w = smk::round_tf32(o.w); }
                    *reinterpret_cast<float4*>(g_out + (size_t)(opix[i] + pix_off) * a.ld_out + col) = o;
                    if constexpr (AFF) {
                        if (a.out2 && mc < (size_t)a.out2_rows) *reinterpret_cast<float4*>(a.out2 + mc * a.ld_out2 + nc) = a.scale2 ? o2 : o;
                    } else {
                        if (EXTRA && a.out2 && mc < (size_t)a.out2_rows) *reinterpret_cast<float4*>(a.out2 + mc * a.ld_out2 + nc) = o;
                    }
                }
            }
            __syncwarp();
        }
    }
}

// ---- reflection halo of a [B, H+2, W+2, C] buffer whose interior has been written -------------------
__global__ void __launch_bounds__(256)
reflect_halo_kernel(float* __restrict__ buf, int B, int H, int W, int C) {
    const int Hp = H + 2, Wp = W + 2, C4 = C >> 2;
    const int halo = 2 * Wp + 2 * H;                       // halo pixels per image
    long total = (long)B * halo * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        int c4 = (int)(i % C4); long t = i / C4; int k = (int)(t % halo); int b = (int)(t / halo);
        int ph, pw;
        if (k < Wp) { ph = 0; pw = k; }
        else if (k < 2 * Wp) { ph = Hp - 1; pw = k - Wp; }
        else { int r = k - 2 * Wp; ph = 1 + (r >> 1); pw = (r & 1) ? Wp - 1 : 0; }
        // ReflectionPad2d(1): padded index p -> interior index |p-1| mirrored at the far edge
        int sh = ph - 1, sw = pw - 1;
        sh = sh < 0 ? 1 : (sh >= H ? H - 2 : sh);
        sw = sw < 0 ? 1 : (sw >= W ? W - 2 : sw);
        const float4* src = reinterpret_cast<const float4*>(buf + (((size_t)b * Hp + sh + 1) * Wp + sw + 1) * C) + c4;
        float4* dst = reinterpret_cast<float4*>(buf + (((size_t)b * Hp + ph) * Wp + pw) * C) + c4;
        *dst = *src;
    }
}

// ---- host: tensor-map encoding through the driver entry points (no link-time libcuda dependency) ------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
struct DriverFns { EncodeTiledFn tiled; EncodeIm2colFn im2col; };

// Resolved once per process (thread-safe static initialisation); null where the driver lacks an entry point.
const DriverFns& driver_fns() {
    static const DriverFns fns = [] {
        auto get = [](const char* name) -> void* {
            void* fn = nullptr;
            cudaDriverEntryPointQueryResult q;
            return cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess ? fn : nullptr;
        };
        return DriverFns{(EncodeTiledFn)get("cuTensorMapEncodeTiled"), (EncodeIm2colFn)get("cuTensorMapEncodeIm2col")};
    }();
    return fns;
}

}  // namespace

int tc_init() {
    SMK_REQUIRE(driver_fns().tiled && driver_fns().im2col, "cuTensorMapEncodeTiled / cuTensorMapEncodeIm2col not available from the driver");
    return 0;
}

int encode_2d(CUtensorMap* map, const float* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, const char* what) {
    if (int rc = tc_init()) return rc;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {ld * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)BK, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = driver_fns().tiled(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, dims, strides, box, estr,
                                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    SMK_REQUIRE(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled failed (%d): rows=%llu cols=%llu ld=%llu box_rows=%u", what, (int)r,
                (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_rows);
    return 0;
}

int encode_nhwc(CUtensorMap* map, const float* base, int B, int H, int W, int C, int ld, int box_w, int box_h, const char* what) {
    if (int rc = tc_init()) return rc;
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)ld * 4, (cuuint64_t)W * ld * 4, (cuuint64_t)H * W * ld * 4};
    cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = driver_fns().tiled(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)base, dims, strides, box, estr,
                                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    SMK_REQUIRE(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled failed (%d): B=%d H=%d W=%d C=%d ld=%d box=%dx%d", what, (int)r,
                B, H, W, C, ld, box_h, box_w);
    return 0;
}

// Lower / upper corner of the 3x3 window per CUTLASS conventions: lower = -pad, upper = pad - (3-1).
int encode_im2col(CUtensorMap* map, const float* base, int B, int H, int W, int C, int ld, int pad, const char* what) {
    if (int rc = tc_init()) return rc;
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)ld * 4, (cuuint64_t)W * ld * 4, (cuuint64_t)H * W * ld * 4};
    int lower[2] = {-pad, -pad};
    int upper[2] = {pad - 2, pad - 2};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = driver_fns().im2col(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)base, dims, strides, lower, upper,
                                     (cuuint32_t)BK, (cuuint32_t)BM, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                     CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    SMK_REQUIRE(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeIm2col failed (%d): B=%d H=%d W=%d C=%d ld=%d pad=%d", what, (int)r,
                B, H, W, C, ld, pad);
    return 0;
}

namespace {

template <int BN, int STAGES, int MINB, bool PERSIST, int X3, bool EXTRA, bool AFF = false>
int launch_kernel(const TcMaps& mp, const TcArgs& a_in, cudaStream_t st, int groups) {
    constexpr size_t stage = X3 ? A_STAGE_BYTES + 2 * BN * BKB : A_STAGE_BYTES + BN * BKB;
    constexpr size_t smem = (size_t)STAGES * stage + (PERSIST ? SLAB_BYTES : 0) + BAR_BYTES + HEAD_PAR_BYTES + 1024;
    static_assert(PERSIST || (size_t)STAGES * stage >= SLAB_BYTES, "single-tile CTAs stage the epilogue in ring stage 0");
    static_assert(MINB * (smem + 1024) <= 228 * 1024, "shared memory budget of MINB resident CTAs");
    SMK_CHECK_CUDA((set_max_dynamic_smem<gemm_tc_kernel<BN, STAGES, MINB, PERSIST, X3, EXTRA, AFF>>((int)smem)));
    TcArgs a = a_in;
    a.tiles_n = cdiv(a.N, BN);
    a.n_tiles_g = cdiv(a.M, BM) * a.tiles_n;
    a.n_tiles = groups * a.n_tiles_g;
    dim3 grid((unsigned)(PERSIST ? std::min(a.n_tiles, MINB * num_sms()) : a.n_tiles));
    SMK_LAUNCH((gemm_tc_kernel<BN, STAGES, MINB, PERSIST, X3, EXTRA, AFF>), dim3(grid), dim3(NUM_THREADS), smem, st, mp, a);
    SMK_CHECK_LAUNCH();
    return 0;
}

template <int BN, int STAGES, int MINB, bool PERSIST, int X3 = 0>
int launch(const TcMaps& mp, const TcArgs& a, cudaStream_t st, int groups) {
    if constexpr (X3 != 2) {                            // X3 = 2 runs plain GEMMs only (tc_conv)
        if constexpr (BN >= 64) {                       // PReLU / second-store affine: N >= 64 (tc_conv checks)
            if (a.prelu || a.scale2) return launch_kernel<BN, STAGES, MINB, PERSIST, X3, true, true>(mp, a, st, groups);
        }
        if (a.mask || a.out2) return launch_kernel<BN, STAGES, MINB, PERSIST, X3, true>(mp, a, st, groups);
    }
    return launch_kernel<BN, STAGES, MINB, PERSIST, X3, false>(mp, a, st, groups);
}

}  // namespace

int tc_conv(const Conv& p, cudaStream_t st, const Conv* p2) {
    if (!p2 && conv3_win_supported(p)) return conv3_win(p, st);       // 224^2 / 112^2, Cout 32 / 64: one patch load per chunk, resident weights
    const int M = p.B * p.H * p.W;
    const int groups = p2 ? 2 : 1;
    SMK_REQUIRE(p.N % 4 == 0 && p.K % 4 == 0 && p.ld_in % 4 == 0 && p.ld_out % 4 == 0, "tc_conv: N, K, ld must be multiples of 4");
    SMK_REQUIRE(p.mode == 0 || (p.Cin % BK == 0 && p.K == 9 * p.Cin), "tc_conv: 3x3 mode needs Cin %% 32 == 0 (got %d)", p.Cin);
    SMK_REQUIRE(p.store != 1 || ((p.N / 4) % 32 == 0), "tc_conv: pixel-shuffle store needs Cout %% 32 == 0");
    SMK_REQUIRE(!p2 || (p2->B == p.B && p2->H == p.H && p2->W == p.W && p2->Cin == p.Cin && p2->N == p.N && p2->K == p.K && p2->mode == p.mode &&
                        p2->relu == p.relu && p2->ld_in == p.ld_in && p2->ld_out == p.ld_out && p2->ld_res == p.ld_res && p2->store == p.store &&
                        p2->res_pad == p.res_pad && p2->round_out == p.round_out && !p2->wgt.wt_lo == !p.wgt.wt_lo && !p2->res == !p.res && p.store != 3),
                "tc_conv: paired problems must have identical shapes and epilogue options");
    int BN = p.N <= 32 ? 32 : (p.N <= 64 ? 64 : 128);
    // Wide 3x3 layers (N a multiple of 256: the generator's 28^2 / 14^2 convolutions, most of its FLOPs): a 128 x 256 tile
    // halves the A-operand bytes wgmma pulls from shared memory per FLOP (TF32 operands are 4 bytes; at BN = 128 the
    // operand reads ask for more than an SM's shared-memory bandwidth).  One persistent CTA per SM, 4-stage ring.
    if (p.mode != 0 && p.N % 256 == 0 && !p.wgt.wt_lo) BN = 256;
    // 3xTF32: plain 1x1 GEMMs (the encoder's 1x1 convs, K <= 960) run X3 = 2; every other problem (3x3 convs, the shuffled
    // store, the mask / second store: the generator's convolutions, K up to 4608; MICA's PReLU / affine epilogues and its
    // K = 25088 fc) X3 = 3, with 64-wide tiles at most.
    const bool plain = p.mode == 0 && p.store == 0 && !p.mask && !p.out2 && !conv_aff(p) && p.K <= 1024;
    const int x3 = !p.wgt.wt_lo ? 0 : plain ? 2 : 3;
    if (x3 == 3) BN = std::min(BN, 64);
    TcMaps mp;
    TcArgs a{};
    a.M = M; a.N = p.N; a.nkb = cdiv(p.K, BK); a.mode = p.mode == 0 ? 0 : 1; a.H = p.H; a.W = p.W;
    a.cpb = p.mode == 0 ? 1 : p.Cin / BK; a.lc = p.mode == 2 ? 0 : -1;
    a.ld_res = p.ld_res; a.res_pad = p.res_pad; a.relu = p.relu;
    a.ld_out = p.ld_out; a.store = p.store; a.round_out = p.round_out;
    a.head_w = p.head_w; a.head_b = p.head_b; a.head_c = p.head_c;
    SMK_REQUIRE(p.store != 3 || (p.N == 32 && p.mode != 0 && p.head_w && p.head_b && p.head_c >= 1 && p.head_c <= 4 && !p.res && !p2),
                "tc_conv: the fused 1x1 head needs a 3x3 conv with N == 32 (one full column tile) and 1..4 head channels");
    SMK_REQUIRE((!p.mask || p.store == 0) && (!p.out2 || p.store != 1) && (!(p.mask || p.out2) || !p2),
                "tc_conv: the mask needs store 0, the second store a non-shuffled store, both a single problem");
    a.mask = p.mask; a.ld_mask = p.ld_mask; a.out2 = p.out2; a.ld_out2 = p.ld_out2; a.out2_rows = p.out2_rows > 0 ? p.out2_rows : M;
    SMK_REQUIRE(!conv_aff(p) || (p.store == 0 && p.N >= 64 && !p2 && (!p.scale2 || (p.bias2 && p.out2))),
                "tc_conv: PReLU / second-store affine need store 0, N >= 64, a single problem, and scale2 with bias2 and out2");
    a.prelu = p.prelu; a.scale2 = p.scale2; a.bias2 = p.bias2; a.round_out2 = p.round_out2;
    for (int g = 0; g < groups; ++g) {
        const Conv& q = g ? *p2 : p;
        a.scale[g] = q.scale; a.bias[g] = q.bias; a.res[g] = q.res; a.out[g] = q.out;
        if (q.mode == 0) {
            if (int rc = encode_2d(&mp.a[g], q.in, (uint64_t)M, (uint64_t)q.K, (uint64_t)q.ld_in, BM, "tc_conv(A)")) return rc;
        } else if (q.mode == 1) {
            if (int rc = encode_im2col(&mp.a[g], q.in, q.B, q.H, q.W, q.Cin, q.ld_in, 1, "tc_conv(A)")) return rc;
        } else {                                            // input buffer is [B, H+2, W+2, C], already reflection padded
            if (int rc = encode_im2col(&mp.a[g], q.in, q.B, q.H + 2, q.W + 2, q.Cin, q.ld_in, 0, "tc_conv(A)")) return rc;
        }
        if (int rc = encode_2d(&mp.b[g], q.wgt.wt, (uint64_t)q.N, (uint64_t)q.K, (uint64_t)q.K, (uint32_t)BN, "tc_conv(W)")) return rc;
        if (q.wgt.wt_lo) { if (int rc = encode_2d(&mp.blo[g], q.wgt.wt_lo, (uint64_t)q.N, (uint64_t)q.K, (uint64_t)q.K, (uint32_t)BN, "tc_conv(W tails)")) return rc; }
        else mp.blo[g] = mp.b[g];
    }
    if (groups == 1) { mp.a[1] = mp.a[0]; mp.b[1] = mp.b[0]; mp.blo[1] = mp.blo[0]; a.scale[1] = a.scale[0]; a.bias[1] = a.bias[0]; a.res[1] = a.res[0]; a.out[1] = a.out[0]; }
    {
        const double cin_eff = p.mode == 0 ? p.K : p.Cin;
        const char* tag = p.tag ? p.tag
                        : p.mode == 0 ? (p.store == 1 ? (p.wgt.wt_lo ? "upconv_gemm_tc3x" : "upconv_gemm_tc") : (p.wgt.wt_lo ? "pw_gemm_tc3x" : "pw_gemm_tc"))
                        : p.store == 3 ? (p.wgt.wt_lo ? "conv3x3_head_gemm_tc3x" : "conv3x3_head_gemm_tc")
                                       : (p.wgt.wt_lo ? "conv3x3_gemm_tc3x" : "conv3x3_gemm_tc");
        if (g_prof_detail) tag = prof_shape_tag(tag, (long)groups * M, p.K, p.N);
        SMK_TAG(tag,
                groups * 4.0 * ((double)M * cin_eff + (double)p.K * p.N + (double)M * p.N * (1 + !!p.res + !!p.mask + !!p.out2) + 2.0 * p.N),
                groups * 2.0 * (double)M * p.N * p.K, st);
    }
    // MINB (third template argument) trades registers for co-resident CTAs: ptxas budgets the 288-thread block as three
    // warpgroups, so MINB = 1 / 2 / 3 cap a thread at 168 / 96 / 72 registers.  At these budgets <256,4,1>, <128,2,2> and
    // <64,2,3> spill (16-220 B) and the 3xTF32 <32,2,3> serialises its wgmmas; spill-free budgets (lower MINB) were measured
    // slower end to end on H100 (fewer CTAs of the concurrent pipeline share an SM), and 128-wide tiles in place of
    // <256,...> much slower, so the spills stay.
    // 3xTF32: fp32-equivalent arithmetic (encoder and generator precision 3).  Every mode and store, one tile per CTA (the fused
    // head loads its constants per CTA); the EXTRA instantiations carry the generator's grad-mode forward and dgrads.
    // X3 = 3 holds BN / 2 more accumulators: one step lower MINB, and 64-wide tiles at most (a 128-wide tile needs more than
    // the 168 registers of MINB = 1 and spills); ptxas: <32, 2, 2> 80 / 77 registers, <64, 2, 1> 132 / 126, no spills.
    if (x3 == 3) {
        if (BN == 32) return launch<32, 2, 2, false, 3>(mp, a, st, groups);
        return launch<64, 2, 1, false, 3>(mp, a, st, groups);
    }
    if (p.wgt.wt_lo) {
        if (BN == 32) return launch<32, 2, 3, false, 2>(mp, a, st, groups);
        if (BN == 64) return launch<64, 2, 2, false, 2>(mp, a, st, groups);
        return launch<128, 2, 1, false, 2>(mp, a, st, groups);
    }
    const long n_tiles = (long)groups * cdiv(M, BM) * cdiv(p.N, BN);
    // 3x3 convolutions (deep K): persistent CTAs for the narrow-N layers and for the few-tile 14x14 layers; the fused head
    // always (its constants are loaded once per CTA).  Everything else runs one tile per CTA with a 2-stage ring: a small
    // footprint, so several CTAs of this kernel — or of the other backbones' and batches' kernels — share an SM and hide
    // each other's prologue / epilogue.
    const bool persist = p.store == 3 || (p.mode != 0 && (BN <= 64 || n_tiles <= 2 * num_sms()));
    if (BN == 256) return launch<256, 4, 1, true>(mp, a, st, groups);
    if (persist) {
        if (BN == 32) return launch<32, 4, 2, true>(mp, a, st, groups);
        if (BN == 64) return launch<64, 3, 2, true>(mp, a, st, groups);
        return a.nkb > 8 ? launch<128, 5, 1, true>(mp, a, st, groups) : launch<128, 2, 2, true>(mp, a, st, groups);
    }
    if (BN == 32) return launch<32, 2, 3, false>(mp, a, st, groups);
    if (BN == 64) return launch<64, 2, 3, false>(mp, a, st, groups);
    return launch<128, 2, 2, false>(mp, a, st, groups);
}

int reflect_halo(float* buf, int B, int H, int W, int C, cudaStream_t st) {
    long total = (long)B * (2 * (W + 2) + 2 * H) * (C / 4);
    SMK_TAG("reflect_halo", 8.0 * (double)total * 4, 0.0, st);
    SMK_LAUNCH(reflect_halo_kernel, dim3((int)std::min<long>((total + 255) / 256, 8L * num_sms())), dim3(256), 0, st, buf, B, H, W, C);
    SMK_CHECK_LAUNCH();
    return 0;
}

}  // namespace smk

// ---- debug / unit-test entry points (tests/test_gpu_kernels.py) -----------------------------------------
extern "C" int smk_debug_conv_tc(const float* in, int ld_in, int B, int H, int W, int Cin, const float* wt, const float* scale,
                                 const float* bias, int N, int K, int mode, int relu, const float* res, int ld_res, int res_pad,
                                 float* out, int ld_out, int store, void* stream) {
    smk::Conv p{};
    p.in = in; p.ld_in = ld_in; p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.wgt = smk::GemmW{nullptr, wt, nullptr}; p.scale = scale; p.bias = bias; p.N = N; p.K = K;
    p.mode = mode; p.relu = relu; p.res = res; p.ld_res = ld_res; p.res_pad = res_pad; p.out = out; p.ld_out = ld_out; p.store = store;
    return smk::tc_conv(p, (cudaStream_t)stream);
}
// 1x1 conv / GEMM on the 3xTF32 path: wt_hi / wt_lo are the TF32 heads and tails of the [N][K] weights.
extern "C" int smk_debug_gemm_tc3x(const float* in, int ld_in, int M, const float* wt_hi, const float* wt_lo, const float* scale,
                                   const float* bias, int N, int K, int relu, const float* res, int ld_res, float* out, int ld_out, void* stream) {
    smk::Conv p{};
    p.in = in; p.ld_in = ld_in; p.B = 1; p.H = 1; p.W = M; p.Cin = K; p.wgt = smk::GemmW{nullptr, wt_hi, wt_lo}; p.scale = scale; p.bias = bias; p.N = N; p.K = K;
    p.mode = 0; p.relu = relu; p.res = res; p.ld_res = ld_res; p.res_pad = 0; p.out = out; p.ld_out = ld_out; p.store = 0; p.round_out = 0;
    return smk::tc_conv(p, (cudaStream_t)stream);
}
// smk_debug_conv_tc on the 3xTF32 path, with every epilogue option of the generator's convolutions: mask [M, ld_mask]
// (zero outputs whose mask <= 0; store 0), out2 [M, ld_out2] (the stored activations again, compact; stores 0, 2, 3) and
// the fused head of store 3 (head_w [N][head_c], head_b [head_c], out [B, head_c, H, W] NCHW, N == 32, 1 <= head_c <= 4).
// Null mask / out2 / head pointers: not used.  Nothing is rounded to TF32.  Each 32-deep k-block is summed apart (X3 = 3),
// except for a plain 1x1 GEMM (mode 0, store 0, no mask / out2), which runs smk_debug_gemm_tc3x's arithmetic.
// A kernel-test entry point: it is exported but not part of include/smirk_b200.h, and tests/test_gpu_generator_x3.py
// declares its argument types itself.
extern "C" int smk_debug_conv_tc3x(const float* in, int ld_in, int B, int H, int W, int Cin, const float* wt_hi, const float* wt_lo,
                                   const float* scale, const float* bias, int N, int K, int mode, int relu, const float* res, int ld_res,
                                   int res_pad, float* out, int ld_out, int store, const float* mask, int ld_mask, float* out2, int ld_out2,
                                   const float* head_w, const float* head_b, int head_c, void* stream) {
    SMK_REQUIRE(wt_hi && wt_lo, "smk_debug_conv_tc3x: the weight heads and tails are both required");
    smk::Conv p{};
    p.in = in; p.ld_in = ld_in; p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.wgt = smk::GemmW{nullptr, wt_hi, wt_lo}; p.scale = scale; p.bias = bias;
    p.N = N; p.K = K; p.mode = mode; p.relu = relu; p.res = res; p.ld_res = ld_res; p.res_pad = res_pad; p.out = out; p.ld_out = ld_out;
    p.store = store; p.round_out = 0; p.mask = mask; p.ld_mask = ld_mask; p.out2 = out2; p.ld_out2 = ld_out2;
    p.head_w = head_w; p.head_b = head_b; p.head_c = head_c;
    return smk::tc_conv(p, (cudaStream_t)stream);
}
extern "C" int smk_debug_reflect_halo(float* buf, int B, int H, int W, int C, void* stream) {
    return smk::reflect_halo(buf, B, H, W, C, (cudaStream_t)stream);
}
