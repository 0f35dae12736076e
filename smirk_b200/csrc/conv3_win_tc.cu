// 3x3 stride-1 convolution for the generator's HIGH-RESOLUTION, NARROW layers (224^2 and 112^2, Cout = 32 / 64;
// reference src/smirk_generator.py:56-60,73-76 -> `_block` :88-119) as a persistent "windowed" TF32 wgmma implicit GEMM.
//
// Why a second 3x3 kernel.  gemm_tc.cu feeds the nine filter taps with nine im2col TMA loads per 32-channel chunk, so
// every input pixel crosses L2 -> shared memory nine times, and every tile re-loads the layer's weights.  For the wide, deep
// layers that hides behind the MMAs.  With Cout = 32 the MMAs are tiny (128 x 32 x 8) and a tile's life is a serial chain of
// short steps.  Here:
//
//   output tile   4 x 30 pixels of one image
//   patch         6 x 32 pixels x 32 channels = 192 rows of 128 bytes, one 4-D tiled TMA box (out-of-image halo zero
//                 filled = the conv's zero padding), SWIZZLE_128B, row r = py * 32 + px — loaded ONCE per channel chunk
//   tap (dy,dx)   A operand = the 128 consecutive patch rows starting at row dy*32 + dx: only the wgmma descriptor's start
//                 address moves (the swizzle follows the absolute shared-memory address, as TMA's does when it writes).
//                 GEMM row m <-> output pixel (m / 32, m % 32); columns 30, 31 of each row wrap into the halo and are not
//                 stored (93.75 % useful rows).
//   weights       [N][9*Cin] K-major; the 9 * Cin/32 boxes of BN x 32 are loaded once per CTA and stay in shared memory
//   two pipelines one CTA per SM runs TWO independent tile pipelines (each: a TMA producer warp and one consumer warpgroup
//                 that issues the wgmmas — two m64 halves of the 128-row tile — and runs the epilogue from its accumulator
//                 registers, a 2-deep patch ring) that share the resident weights, so one pipeline's loads and epilogue
//                 overlap the other's MMAs.
// L2 -> SM traffic per output pixel drops from 9 x 128 B (+ the weights again for every tile) to 1.6 x 128 B.
// Epilogue as in gemm_tc.cu (folded BN, ReLU, TF32 rounding, coalesced NHWC stores) plus the fused 1x1 head + sigmoid of
// the network's last layer (store 3).
#include "gemm_tc.cuh"
#include "tc_ptx.cuh"

namespace smk {
namespace {

using namespace ptx;

constexpr int PIPES = 2;
constexpr int NUM_THREADS = PIPES * 128 + PIPES * 32;   // warps 0..7: consumer warpgroups (pipeline = warp / 4); warps 8, 9: TMA producers
constexpr int PW = 32, TH = 4, TW = 30;              // patch width, output tile height / width
constexpr int PATCH_BYTES = (TH + 2) * PW * 128;     // 24 KiB
constexpr int STAGES = 2;                            // patch ring depth per pipeline
constexpr int SLAB_BYTES = 4 * 2048;                 // per pipeline: 16 rows x 128 B per consumer warp
constexpr int TAIL_BYTES = 1024;                     // the last tap view reads 2 rows past its patch: keep that inside the allocation
constexpr int PIPE_BYTES = STAGES * PATCH_BYTES + TAIL_BYTES + SLAB_BYTES;      // 58 368 B
constexpr int NB = 4;                                // weight-ring depth per pipeline (layers whose weights do not fit resident)
constexpr int BAR_BYTES = 512;
constexpr int HEAD_PAR_BYTES = 1088;                 // per pipeline, store 3: [32][8] per-channel constants + 4 head biases

struct WinArgs {
    int H, W, N;
    int nchunks;                 // Cin / 32
    int tiles_x, tiles_y, n_tiles;
    const float* scale; const float* bias;
    int relu, round_out;
    float* out; int ld_out;
    int store;                   // 0 plain NHWC, 3 fused 1x1 head + sigmoid (NCHW)
    const float* head_w; const float* head_b; int head_c;
    const float* mask; int ld_mask;   // store 0: zero outputs whose mask[pixel, n] <= 0 (ReLU backward)
    float* out2; int ld_out2;         // the stored activations again, compact NHWC (store 3: the activations it does not store)
    int out2_rows;                    // out2 takes the pixels m < out2_rows
};

// RES = true : the layer's whole weight matrix stays in shared memory, shared by both pipelines (<= 72 KB);
// RES = false: each pipeline streams the (chunk, tap) weight boxes through its own NB-deep ring (the 112^2 Cout-64 layers with
//              147 - 295 KB of weights): the input window is still loaded once per chunk instead of nine times.
// EXTRA = true: the epilogue also applies `mask` and writes `out2` (backward / grad-mode forward); the forward-only
//               instantiations are compiled without them.
template <int BN, bool RES, bool EXTRA>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv3_win_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const WinArgs a) {
    constexpr int B_BYTES = BN * 128;                      // one (chunk, tap) weight box
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool producer = warp >= PIPES * 4;
    const int pipe = producer ? warp - PIPES * 4 : warp >> 2;      // pipeline of this warp
    uint8_t* sP = smem + pipe * PIPE_BYTES;                // this pipeline's patch ring (+ tail) ...
    uint8_t* slabs = sP + STAGES * PATCH_BYTES + TAIL_BYTES;      // ... and epilogue staging
    // weights: resident [chunk][tap][BN x 128 B] shared by both pipelines, or one NB-deep ring of boxes per pipeline
    const int w_bytes = RES ? a.nchunks * 9 * B_BYTES : PIPES * NB * B_BYTES;
    uint8_t* sW = smem + PIPES * PIPE_BYTES + (RES ? 0 : pipe * NB * B_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + PIPES * PIPE_BYTES + w_bytes);
    constexpr int PER_PIPE_BARS = 2 * STAGES + 2 * NB;
    uint64_t* w_full = bars;                               // [1]
    uint64_t* p_full = bars + 1 + pipe * PER_PIPE_BARS;    // per pipeline: p_full[STAGES], p_empty[STAGES], b_full[NB], b_empty[NB]
    uint64_t* p_empty = p_full + STAGES;
    uint64_t* b_full = p_empty + STAGES;
    uint64_t* b_empty = b_full + NB;
    float* hpar = reinterpret_cast<float*>(smem + PIPES * PIPE_BYTES + w_bytes + BAR_BYTES + pipe * HEAD_PAR_BYTES);

    if (producer && lane == 0) {
        if (pipe == 0) { prefetch_tensormap(&tmX); prefetch_tensormap(&tmW); mbar_init(w_full, 1); }
        for (int s = 0; s < STAGES; ++s) { mbar_init(&p_full[s], 1); mbar_init(&p_empty[s], 4); }
        for (int i = 0; i < NB; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], 4); }
        fence_barrier_init();
    }
    __syncthreads();

    auto decode = [&](int t, int& img, int& h0, int& w0) {
        const int tx = t % a.tiles_x; t /= a.tiles_x;
        const int ty = t % a.tiles_y; img = t / a.tiles_y;
        h0 = ty * TH; w0 = tx * TW;
    };
    // tiles are strided over (CTA, pipeline) pairs
    const int t_first = blockIdx.x * PIPES + pipe, t_step = gridDim.x * PIPES;

    if (producer) {
        if (lane == 0) {
            // ===== TMA producer: (pipeline 0) the weights once; then one patch per (tile, channel chunk) =====
            if (RES && pipe == 0) {
                mbar_expect_tx(w_full, (uint32_t)w_bytes);
                for (int c = 0; c < a.nchunks; ++c)
                    for (int tap = 0; tap < 9; ++tap)
                        tma_load_2d(&tmW, sW + (c * 9 + tap) * B_BYTES, w_full, tap * a.nchunks * 32 + c * 32, 0);
            }
            int it = 0, itb = 0;
            for (int t = t_first; t < a.n_tiles; t += t_step) {
                int img, h0, w0;
                decode(t, img, h0, w0);
                for (int c = 0; c < a.nchunks; ++c, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(&p_empty[s], ((uint32_t)(it / STAGES) & 1u) ^ 1u);
                    mbar_expect_tx(&p_full[s], (uint32_t)PATCH_BYTES);
                    tma_load_4d(&tmX, sP + s * PATCH_BYTES, &p_full[s], c * 32, w0 - 1, h0 - 1, img);
                    if (!RES) {
                        for (int tap = 0; tap < 9; ++tap, ++itb) {
                            const int sb = itb % NB;
                            mbar_wait(&b_empty[sb], ((uint32_t)(itb / NB) & 1u) ^ 1u);
                            mbar_expect_tx(&b_full[sb], (uint32_t)B_BYTES);
                            tma_load_2d(&tmW, sW + sb * B_BYTES, &b_full[sb], tap * a.nchunks * 32 + c * 32, 0);
                        }
                    }
                }
            }
        }
        return;
    }

    // ===== consumer warpgroup of this pipeline: MMAs, then the epilogue from the accumulator registers =====
    const int wq = warp & 3;
    uint8_t* slab = slabs + wq * 2048;
    const int sub = lane >> 3, jj = lane & 7;
    if (BN == 32 && a.store == 3) {                      // head constants of channel `lane` (see gemm_tc.cu)
        if (wq == 0) {
            hpar[lane * 8 + 0] = __ldg(a.scale + lane); hpar[lane * 8 + 1] = __ldg(a.bias + lane);
#pragma unroll
            for (int co = 0; co < 4; ++co) hpar[lane * 8 + 2 + co] = co < a.head_c ? __ldg(a.head_w + (size_t)lane * a.head_c + co) : 0.f;
            if (lane < 4) hpar[256 + lane] = lane < a.head_c ? __ldg(a.head_b + lane) : 0.f;
        }
        named_barrier(1 + pipe, 128);
    }
    if (RES) mbar_wait(w_full, 0);
    const uint32_t w_base = smem_u32(sW);
    int it = 0, itb = 0;
    for (int t = t_first; t < a.n_tiles; t += t_step) {
        int img, h0, w0;
        decode(t, img, h0, w0);
        float acc[2][BN / 2];
#pragma unroll
        for (int mb = 0; mb < 2; ++mb)
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[mb][i] = 0.f;
        for (int c = 0; c < a.nchunks; ++c, ++it) {
            const int s = it % STAGES;
            mbar_wait(&p_full[s], (uint32_t)(it / STAGES) & 1u);
            const uint32_t p_base = smem_u32(sP + s * PATCH_BYTES);
#pragma unroll
            for (int tap = 0; tap < 9; ++tap) {
                const uint32_t a_tap = p_base + (uint32_t)(((tap / 3) * PW + (tap % 3)) * 128);
                uint32_t b_tap;
                int sb = 0;
                if (RES) {
                    b_tap = w_base + (uint32_t)((c * 9 + tap) * B_BYTES);
                } else {
                    sb = itb % NB;
                    mbar_wait(&b_full[sb], (uint32_t)(itb / NB) & 1u);
                    b_tap = w_base + (uint32_t)(sb * B_BYTES);
                    ++itb;
                }
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k)
#pragma unroll
                    for (int mb = 0; mb < 2; ++mb)
                        Wgmma<BN>::ss(acc[mb], make_smem_desc(a_tap + mb * 64 * 128 + k * 32), make_smem_desc(b_tap + k * 32), 1u);
                wgmma_commit();
                if (!RES) {                                  // the weight box may be overwritten once these MMAs have read it
                    wgmma_wait<0>();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&b_empty[sb]);
                }
            }
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&p_empty[s]);         // the patch may be overwritten
        }
#pragma unroll
        for (int mb = 0; mb < 2; ++mb) {
            const int mrow = mb * 64 + wq * 16;              // first tile row of this warp's slab
#pragma unroll
            for (int c0 = 0; c0 < BN; c0 += 32) {
                stage32<BN>(slab, acc[mb], c0, lane);
                __syncwarp();
                if (BN == 32 && a.store == 3) {
                    // fused 1x1 head + sigmoid (smirk_generator.py:77-78 -> :86), N == BN == 32: lane r < 16 = slab row r = one
                    // pixel with all 32 accumulators; constants by broadcast LDS; NCHW stores
                    const int m = mrow + lane, oy = m / PW, ox = m - oy * PW;
                    const int oh = h0 + oy, ow = w0 + ox;
                    if (lane < 16 && ox < TW && oh < a.H && ow < a.W) {
                        float a0 = hpar[256], a1 = hpar[257], a2 = hpar[258], a3 = hpar[259];
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
                            const size_t px = (size_t)(img * a.H + oh) * a.W + ow;
                            if (EXTRA && a.out2 && px < (size_t)a.out2_rows)
                                *reinterpret_cast<float4*>(a.out2 + px * a.ld_out2 + 4 * j) = make_float4(xs[0], xs[1], xs[2], xs[3]);
                        }
                        const int hw_px = a.H * a.W;
                        float* dst = a.out + (size_t)img * a.head_c * hw_px + (size_t)oh * a.W + ow;
                        dst[0] = 1.f / (1.f + __expf(-a0));
                        if (a.head_c > 1) dst[hw_px] = 1.f / (1.f + __expf(-a1));
                        if (a.head_c > 2) dst[2 * (size_t)hw_px] = 1.f / (1.f + __expf(-a2));
                        if (a.head_c > 3) dst[3 * (size_t)hw_px] = 1.f / (1.f + __expf(-a3));
                    }
                    __syncwarp();
                    continue;
                }
                const int nc = c0 + jj * 4;
                if (nc < a.N) {
                    const float4 sc = __ldg(reinterpret_cast<const float4*>(a.scale + nc));
                    const float4 bi = __ldg(reinterpret_cast<const float4*>(a.bias + nc));
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int r = 4 * i + sub;
                        const int m = mrow + r, oy = m / PW, ox = m - oy * PW;
                        const int oh = h0 + oy, ow = w0 + ox;
                        if (!(ox < TW && oh < a.H && ow < a.W)) continue;
                        const float4 x = slab_chunk(slab, r, jj);
                        float4 o;
                        o.x = fmaf(x.x, sc.x, bi.x); o.y = fmaf(x.y, sc.y, bi.y); o.z = fmaf(x.z, sc.z, bi.z); o.w = fmaf(x.w, sc.w, bi.w);
                        if (a.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
                        const size_t pix = (size_t)(img * a.H + oh) * a.W + ow;
                        if (EXTRA && a.mask) {
                            const float4 k4 = __ldg(reinterpret_cast<const float4*>(a.mask + pix * a.ld_mask + nc));
                            o.x = k4.x > 0.f ? o.x : 0.f; o.y = k4.y > 0.f ? o.y : 0.f; o.z = k4.z > 0.f ? o.z : 0.f; o.w = k4.w > 0.f ? o.w : 0.f;
                        }
                        if (a.round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
                        *reinterpret_cast<float4*>(a.out + pix * a.ld_out + nc) = o;
                        if (EXTRA && a.out2 && pix < (size_t)a.out2_rows) *reinterpret_cast<float4*>(a.out2 + pix * a.ld_out2 + nc) = o;
                    }
                }
                __syncwarp();
            }
        }
    }
}

size_t win_smem_bytes(int nchunks, int BN, bool res) {
    return (size_t)PIPES * PIPE_BYTES + (res ? (size_t)nchunks * 9 * BN * 128 : (size_t)PIPES * NB * BN * 128) + BAR_BYTES + PIPES * HEAD_PAR_BYTES + 1024;
}
bool win_resident(int nchunks, int BN) { return win_smem_bytes(nchunks, BN, true) <= 227 * 1024; }

template <int BN, bool RES, bool EXTRA>
int launch_kernel(const CUtensorMap& tmX, const CUtensorMap& tmW, const WinArgs& a, cudaStream_t st) {
    const size_t smem = win_smem_bytes(a.nchunks, BN, RES);
    SMK_REQUIRE(smem <= 227 * 1024, "conv3_win: shared-memory budget exceeded (%zu bytes)", smem);
    SMK_CHECK_CUDA((set_max_dynamic_smem<conv3_win_kernel<BN, RES, EXTRA>>(227 * 1024)));
    SMK_LAUNCH((conv3_win_kernel<BN, RES, EXTRA>), dim3((unsigned)std::min(cdiv(a.n_tiles, PIPES), num_sms())), dim3(NUM_THREADS), smem, st, tmX, tmW, a);
    SMK_CHECK_LAUNCH();
    return 0;
}

template <int BN, bool RES>
int launch(const CUtensorMap& tmX, const CUtensorMap& tmW, const WinArgs& a, cudaStream_t st) {
    if (a.mask || a.out2) return launch_kernel<BN, RES, true>(tmX, tmW, a, st);
    return launch_kernel<BN, RES, false>(tmX, tmW, a, st);
}

}  // namespace

bool conv3_win_supported(const Conv& p) {
    if (p.mode != 1 || p.res || p.wgt.wt_lo || (p.store != 0 && p.store != 3) || (p.store == 3 && (p.N != 32 || p.mask))) return false;
    if (p.Cin % 32 != 0 || p.K != 9 * p.Cin || (p.N != 32 && p.N != 64)) return false;
    return p.W >= 56;                                             // low-resolution layers are MMA-bound: gemm_tc's wide tiles win there
}

// mode 1 (3x3, zero padding 1), store 0 or 3, no residual.
int conv3_win(const Conv& p, cudaStream_t st) {
    SMK_REQUIRE(conv3_win_supported(p), "conv3_win: unsupported problem (needs 3x3 zero-pad, Cin %% 32 == 0, N in {32, 64}, W >= 56)");
    SMK_REQUIRE(p.N % 4 == 0 && p.ld_in % 4 == 0 && p.ld_out % 4 == 0, "conv3_win: N and strides must be multiples of 4");
    SMK_REQUIRE(p.store != 3 || (p.N == 32 && p.head_w && p.head_b && p.head_c >= 1 && p.head_c <= 4), "conv3_win: the fused head needs N == 32");
    const int BN = p.N <= 32 ? 32 : 64;
    CUtensorMap tmX, tmW;
    if (int rc = encode_nhwc(&tmX, p.in, p.B, p.H, p.W, p.Cin, p.ld_in, PW, TH + 2, "conv3_win(x)")) return rc;
    if (int rc = encode_2d(&tmW, p.wgt.wt, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)p.K, (uint32_t)BN, "conv3_win(w)")) return rc;
    WinArgs a{};
    a.H = p.H; a.W = p.W; a.N = p.N; a.nchunks = p.Cin / 32;
    a.tiles_x = cdiv(p.W, TW); a.tiles_y = cdiv(p.H, TH); a.n_tiles = a.tiles_x * a.tiles_y * p.B;
    a.scale = p.scale; a.bias = p.bias; a.relu = p.relu; a.round_out = p.round_out;
    a.out = p.out; a.ld_out = p.ld_out; a.store = p.store; a.head_w = p.head_w; a.head_b = p.head_b; a.head_c = p.head_c;
    a.mask = p.mask; a.ld_mask = p.ld_mask; a.out2 = p.out2; a.ld_out2 = p.ld_out2;
    a.out2_rows = p.out2_rows > 0 ? p.out2_rows : p.B * p.H * p.W;
    {
        const double M = (double)p.B * p.H * p.W;
        const char* tag = p.tag ? p.tag : p.store == 3 ? "conv3x3_win_head_tc" : "conv3x3_win_tc";
        if (g_prof_detail) tag = prof_shape_tag(tag, (long)M, p.K, p.N);
        SMK_TAG(tag, 4.0 * (M * p.Cin + (double)p.K * p.N + M * (p.store == 3 ? p.head_c : p.N) + M * p.N * (!!p.mask + !!p.out2) + 2.0 * p.N),
                2.0 * M * p.N * p.K, st);
    }
    // resident weights: 36 KB (32->32), 72 KB (64->32, 32->64); larger layers stream them through a ring
    if (win_resident(a.nchunks, BN)) return BN == 32 ? launch<32, true>(tmX, tmW, a, st) : launch<64, true>(tmX, tmW, a, st);
    return BN == 32 ? launch<32, false>(tmX, tmW, a, st) : launch<64, false>(tmX, tmW, a, st);
}

}  // namespace smk

extern "C" int smk_debug_conv3_win(const float* in, int ld_in, int B, int H, int W, int Cin, const float* wt, const float* scale,
                                   const float* bias, int N, int relu, float* out, int ld_out, void* stream) {
    smk::Conv p{};
    p.in = in; p.ld_in = ld_in; p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.wgt = smk::GemmW{nullptr, wt, nullptr}; p.scale = scale; p.bias = bias; p.N = N; p.K = 9 * Cin;
    p.mode = 1; p.relu = relu; p.out = out; p.ld_out = ld_out; p.store = 0;
    return smk::conv3_win(p, (cudaStream_t)stream);
}
