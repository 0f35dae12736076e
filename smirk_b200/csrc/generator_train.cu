// SmirkGenerator in train mode: BatchNorm over batch statistics (with the running-statistics update) and the gradients of
// every parameter, for the reference trainer's generator steps (src/smirk_trainer.py:94,295 with base_trainer.py:108-111's
// .train()).
//
// A train handle holds the topology only (gen::TrainTopo).  Every call reads the module's current parameters through device
// pointers (SmkGeneratorTrainArgs) and repacks the weights into the workspace (trn::pack), so an optimizer step needs no
// new handle.  The forward walks the UNet front to back as generator_forward does, on the same smk::conv kernels, but with
// BN unfolded: per 3x3 conv the pre-BN output z (unit scale, zero bias), then trn::bn_forward (fixed-chunk fp64 statistics,
// running statistics, apply + ReLU / residual, written into a concat slice or a padded buffer where the next layer wants
// it).  Reflection padding: mode 2 over the unpadded input at precision 0; at precisions 1 and 3 a padded copy whose halo
// reflect_halo fills.  The 1x1 head runs after the last BatchNorm (conv1x1_sigmoid_nchw) at every precision.
// The backward walks back to front as smk_generator_backward does, with the same dgrad helpers (gen::) over weights packed
// without a BN scale, and per layer trn::bn_backward and a weight gradient: conv3_wgrad below for the 3x3 convs (fp32
// CUDA cores, split K over fixed pixel chunks, fixed-order reduce), trn::pw_wgrad over the dgrad's space-to-depth copy for
// the up-convolutions and over the head's input for the head.  No atomics: results are bitwise reproducible, and every call
// is CUDA-graph capturable.
#include "nn_kernels.cuh"
#include "gemm_tc.cuh"
#include "generator.cuh"
#include "train_common.cuh"
#include "../../include/smirk_b200_generator_train.h"

using namespace trn;
using gen::TrainConv;
using gen::TrainTopo;
using gen::TrainUp;
using smk::cdiv;
using smk::grid_of;

namespace {

// 3x3 conv weight gradient, split K: part[chunk][co][ci][tap] (torch's layout) = sum over the chunk's pixels p of
// g[p][co] * A(p, tap, ci), A the conv's input a [B,H,W,lda] (its first cin channels) at pixel p + tap offset, with zero
// padding (refl 0) or reflection padding (refl 1) — the unpadded input, mirrored in the loader.  GEMM view: rows co, columns
// k = tap * cin + ci; a 64 x 64 tile per CTA, 16 pixels per step, 4 x 4 outputs per thread (pw_wgrad's scheme).
__global__ void __launch_bounds__(256)
conv3_wgrad_kernel(const float* __restrict__ g, const float* __restrict__ a, int lda, int B, int H, int W, int cin, int Co, int refl, long chunk,
                   float* __restrict__ part) {
    __shared__ float gs[16][64], as[16][64];
    const int K = 9 * cin;
    const int k0 = blockIdx.x * 64, co0 = blockIdx.y * 64, tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;
    const long M = (long)B * H * W, p0 = blockIdx.z * chunk, p1 = min(M, p0 + chunk);
    const int col = tid % 64, row0 = tid / 64;          // this thread's loads: column col, rows row0 + 4 r
    const int kk = k0 + col, tap = kk / cin, ci = kk - tap * cin, dy = tap / 3 - 1, dx = tap % 3 - 1;
    const bool kok = kk < K, cok = co0 + col < Co;
    float acc[4][4] = {};
    for (long pb = p0; pb < p1; pb += 16) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int row = row0 + 4 * r;
            const long p = pb + row;
            const bool ok = p < p1;
            gs[row][col] = ok && cok ? __ldg(g + (size_t)p * Co + co0 + col) : 0.f;
            float v = 0.f;
            if (ok && kok) {
                const int w = (int)(p % W); const long t = p / W; const int h = (int)(t % H); const long b = t / H;
                int iy = h + dy, ix = w + dx;
                if (refl) {
                    iy = iy < 0 ? 1 : (iy >= H ? H - 2 : iy);
                    ix = ix < 0 ? 1 : (ix >= W ? W - 2 : ix);
                }
                if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(a + ((size_t)(b * H + iy) * W + ix) * lda + ci);
            }
            as[row][col] = v;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            float gv[4], av[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) { gv[j] = gs[k][ty * 4 + j]; av[j] = as[k][tx * 4 + j]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(gv[i], av[j], acc[i][j]);
        }
        __syncthreads();
    }
    float* out = part + (size_t)blockIdx.z * Co * K;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int k = k0 + tx * 4 + j;
        if (k >= K) continue;
        const int tp = k / cin, c = k - tp * cin;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int co = co0 + ty * 4 + i;
            if (co < Co) out[((size_t)co * cin + c) * 9 + tp] = acc[i][j];
        }
    }
}

// The head's pre-sigmoid gradient, NCHW g_y / y [B,cout,HW] -> NHWC t [B*HW, cout]: t = g_y * y (1 - y).
__global__ void __launch_bounds__(256)
sigmoid_bwd_kernel(const float* __restrict__ gy, const float* __restrict__ y, int B, int HW, int cout, float* __restrict__ t) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * HW * cout) return;
    const int j = (int)(i % cout); const long pix = i / cout;
    const int b = (int)(pix / HW), r = (int)(pix - (long)b * HW);
    const size_t o = ((size_t)b * cout + j) * HW + r;
    const float yv = __ldg(y + o);
    t[i] = __ldg(gy + o) * (yv * (1.f - yv));
}

// pw_wgrad's [cin][q * cout + o] -> torch's ConvTranspose2d layout [cin][cout][2][2] (q = dy * 2 + dx).
__global__ void __launch_bounds__(256)
upconv_wgrad_order_kernel(const float* __restrict__ in, int cin, int cout, float* __restrict__ out) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)cin * cout * 4) return;
    const int q = (int)(i % 4); const long t = i / 4; const int o = (int)(t % cout); const long c = t / cout;
    out[i] = in[(size_t)c * 4 * cout + (size_t)q * cout + o];
}

// The 3x3 weight gradient from g [B,H,W,cout] (gradient of the conv's output) and its input a (pixel stride lda, first cin
// channels): split K over wgrad_chunks(...) chunks of pixels; with one chunk the kernel writes out directly.
int conv3_wgrad(const float* g, const float* a, int lda, int B, int H, int W, int cin, int cout, bool refl, float* part, float* out,
                cudaStream_t st) {
    const long M = (long)B * H * W, K = 9L * cin;
    const long tiles = (long)cdiv(K, 64) * cdiv(cout, 64);
    const int nch = wgrad_chunks(M, tiles, 64 * 64, 512);
    const long chunk = cdiv(M, nch);
    SMK_TAG("conv3_wgrad", 4.0 * M * (cout + 9.0 * cin) + 4.0 * nch * cout * K, 2.0 * M * cout * K, st);
    SMK_LAUNCH(conv3_wgrad_kernel, dim3(cdiv(K, 64), cdiv(cout, 64), nch), dim3(256), 0, st, g, a, lda, B, H, W, cin, cout, refl ? 1 : 0, chunk,
               nch == 1 ? out : part);
    SMK_CHECK_LAUNCH();
    return nch == 1 ? 0 : sum_chunks(part, nch, (long)cout * K, out, st);
}

// ---- host side ----------------------------------------------------------------------------------------------------------

// Calls fn(conv) for every 3x3 conv of the topology.
template <typename Fn>
void each_conv(const TrainTopo& T, Fn&& fn) {
    for (int l = 0; l < 5; ++l) for (int j = 0; j < 2; ++j) fn(T.enc[l][j]);
    for (const TrainConv& c : T.res) fn(c);
    for (int l = 0; l < 4; ++l) for (int j = 0; j < 2; ++j) fn(T.dec[l][j]);
}

// Floats of the largest up-convolution weight, [cin][4 cout].
size_t up_floats(const SmkGenerator* h) { return (size_t)16 * h->f * 4 * 8 * h->f; }

// Floats of one copy of the per-call packed weights: every 3x3 conv and up-convolution (forward or dgrad: the same size),
// plus the up-convolutions' replicated biases and the head's [f][cout] weights.
size_t packed_floats(const SmkGenerator* h) {
    const TrainTopo& T = h->topo;
    size_t n = (size_t)h->f * h->cout;
    each_conv(T, [&](const TrainConv& c) { n += (size_t)9 * c.cin_p * c.cout; });
    for (int l = 0; l < 4; ++l) n += (size_t)T.up[l].cin * 4 * T.up[l].cout + 4 * T.up[l].cout;
    return n;
}

// Workspace plan (floats unless noted); forward and backward carve it alike, so one size serves both.
struct Ws {
    float* pk; double2* part; float* gb; float* wpart; float* upw;          // packed weights, BN partials, wgrad partials / reorder
    float* pad[4];                                                            // [B,16,16,16f]: forward (tc) / backward ResNet stream
    float* g[2]; float* gcat[4]; float* s2d;                                  // backward activation gradients
};
size_t ws_bytes(const SmkGenerator* h, int B) {
    const size_t f = h->f, cb = 16 * f;
    size_t n = smk::ws_round(packed_floats(h) * (h->precision == 3 ? 2 : 1) * 4) + smk::ws_round((size_t)kMaxChunks * cb * 16) +
               smk::ws_round(2 * cb * 4) + smk::ws_round(kWgradPart * 4) + smk::ws_round(up_floats(h) * 4) + 4 * smk::ws_round((size_t)B * 256 * cb * 4);
    n += 2 * smk::ws_round((size_t)B * 224 * 224 * std::max<size_t>(f, h->cin_p) * 4);
    for (int l = 0; l < 4; ++l) n += smk::ws_round((size_t)B * (224 >> l) * (224 >> l) * 2 * (f << l) * 4);
    n += smk::ws_round((size_t)B * 112 * 112 * 4 * f * 4);
    return n;
}
bool carve(smk::Workspace& w, const SmkGenerator* h, int B, Ws* o) {
    const size_t f = h->f, cb = 16 * f;
    o->pk = w.take<float>(packed_floats(h) * (h->precision == 3 ? 2 : 1));
    o->part = w.take<double2>((size_t)kMaxChunks * cb);
    o->gb = w.take<float>(2 * cb);
    o->wpart = w.take<float>(kWgradPart);
    o->upw = w.take<float>(up_floats(h));
    for (int i = 0; i < 4; ++i) o->pad[i] = w.take<float>((size_t)B * 256 * cb);
    for (int i = 0; i < 2; ++i) o->g[i] = w.take<float>((size_t)B * 224 * 224 * std::max<size_t>(f, h->cin_p));
    for (int l = 0; l < 4; ++l) o->gcat[l] = w.take<float>((size_t)B * (224 >> l) * (224 >> l) * 2 * (f << l));
    o->s2d = w.take<float>((size_t)B * 112 * 112 * 4 * f);
    return o->s2d != nullptr;
}

// The packed weights of one call: per 3x3 conv and up-convolution its operand (forward or dgrad), the up-convolutions'
// biases replicated over the four sub-positions (forward), and the head's weights as [f][cout].
struct Packed { std::vector<smk::GemmW> enc, res, dec, up; std::vector<const float*> up_bias; const float* head_w = nullptr; };

int pack_weights(const SmkGenerator* h, const SmkGeneratorTrainArgs* a, bool dgrad, float* dst, Packed* P, cudaStream_t st) {
    const TrainTopo& T = h->topo;
    const bool tc = h->precision != 0, x3 = h->precision == 3;
    std::vector<PackJob> jobs;
    auto add = [&](PackJob j, bool split) -> smk::GemmW {
        j.split = split ? 1 : 0;
        const size_t n = pack_floats(j);
        j.hi = dst; j.lo = split && x3 ? dst + n : nullptr;
        dst += n * (j.lo ? 2 : 1);
        jobs.push_back(j);
        return split ? smk::GemmW{nullptr, j.hi, j.lo} : smk::GemmW{j.hi, nullptr, nullptr};
    };
    auto c3 = [&](const TrainConv& c) {
        PackJob j{};
        j.kind = dgrad ? CONV3_DGRAD : CONV3_FWD; j.src = a->tensors[c.t]; j.cin = c.cin; j.cin_p = c.cin_p; j.cout = c.cout;
        return add(j, tc);
    };
    P->enc.clear(); P->res.clear(); P->dec.clear(); P->up.clear(); P->up_bias.clear();
    for (int l = 0; l < 5; ++l) for (int k = 0; k < 2; ++k) P->enc.push_back(c3(T.enc[l][k]));
    for (const TrainConv& c : T.res) P->res.push_back(c3(c));
    for (int l = 0; l < 4; ++l) {
        PackJob j{};
        j.kind = dgrad ? UP_DGRAD : UP_FWD; j.src = a->tensors[T.up[l].t]; j.cin = T.up[l].cin; j.cout = T.up[l].cout;
        P->up.push_back(add(j, tc));
        if (!dgrad) {
            PackJob b{};
            b.kind = UP_BIAS; b.src = a->tensors[T.up[l].t + 1]; b.cout = T.up[l].cout;
            P->up_bias.push_back(add(b, false).w);
        }
        for (int k = 0; k < 2; ++k) P->dec.push_back(c3(T.dec[l][k]));
    }
    PackJob j{};                                           // head [cout][f] -> [f][cout]
    j.kind = MAT; j.src = a->tensors[T.head_t]; j.rows = h->cout; j.cols = h->f; j.transpose = 1;
    P->head_w = add(j, false).w;
    return pack(jobs, 8.0 * packed_floats(h) * (x3 ? 1.5 : 1.0), st);
}

BnRef bn_ref(const SmkGeneratorTrainArgs* a, const SmkGeneratorTrainGrads* gr, const TrainConv& c) {
    BnRef r{};
    float* const* t = a->tensors;
    r.w = t[c.t]; r.gamma = t[c.t + 1]; r.beta = t[c.t + 2]; r.rmean = t[c.t + 3]; r.rvar = t[c.t + 4];
    r.nbt = (long long*)a->num_batches_tracked[c.bn];
    if (gr && gr->tensors) { r.gw = gr->tensors[c.t]; r.ggamma = gr->tensors[c.t + 1]; r.gbeta = gr->tensors[c.t + 2]; }
    return r;
}

// One train-mode 3x3 conv: z = conv(in) with unit scale and zero bias (pre-BN).  At precisions 1 and 3 a reflection-padded
// conv's `in` is the padded buffer.
int conv3(const SmkGenerator* h, const smk::GemmW& w, const TrainConv& c, const float* in, int ld_in, int B, float* z, cudaStream_t st) {
    smk::Conv p{};
    p.in = in; p.ld_in = ld_in; p.B = B; p.H = c.S; p.W = c.S; p.Cin = c.cin_p; p.wgt = w; p.scale = h->ones; p.bias = h->zeros;
    p.N = c.cout; p.K = 9 * c.cin_p; p.mode = c.refl ? 2 : 1; p.out = z; p.ld_out = c.cout;
    return smk::conv(p, st);
}

// Topology of a train handle: the layers with their tensor and BatchNorm indices, the saved layout and the statistics.
void build_topology(SmkGenerator* h) {
    TrainTopo& T = h->topo;
    const int f = h->f;
    int t = 0, bn = 0;
    auto add = [&](const std::string& n, int S, int C) { return h->saved.add(n, S, S, C); };
    auto conv = [&](int cin, int cin_p, int cout, int S, bool refl, const std::string& zname, const std::string& yname) {
        TrainConv c;
        c.t = t; c.bn = bn++; c.cin = cin; c.cin_p = cin_p; c.cout = cout; c.S = S; c.refl = refl;
        t += 5;
        c.sv_z = add(zname, S, cout);
        c.sv_y = yname.empty() ? -1 : add(yname, S, cout);
        c.stats = T.stats_floats; T.stats_floats += 2 * (size_t)cout;
        return c;
    };
    T.sv_input = add("input", 224, h->cin_p);
    int c_in = h->cin, c_in_p = h->cin_p;
    for (int l = 0; l < 4; ++l) {
        const int S = 224 >> l, c = f << l;
        const std::string e = "enc" + std::to_string(l + 1);
        T.enc[l][0] = conv(c_in, c_in_p, c, S, false, e + "conv1", e + "norm1");
        T.enc[l][1] = conv(c, c, c, S, false, e + "conv2", "");            // its output: the skip half of the decoder's input
        T.sv_cat[l] = add("dec" + std::to_string(l + 1) + "cat", S, 2 * c);
        T.sv_pool[l] = add("pool" + std::to_string(l + 1), S / 2, c);
        c_in = c_in_p = c;
    }
    const int cb = 16 * f;
    T.enc[4][0] = conv(8 * f, 8 * f, cb, 14, false, "bottleneckconv1", "bottlenecknorm1");
    T.enc[4][1] = conv(cb, cb, cb, 14, false, "bottleneckconv2", "bottlenecknorm2");
    T.res.clear();
    for (int r = 0; r < h->nres; ++r) {
        const std::string n = "res" + std::to_string(r);
        T.res.push_back(conv(cb, cb, cb, 14, true, n + "conv1", n + "norm1"));
        T.res.push_back(conv(cb, cb, cb, 14, true, n + "conv2", n + "norm2"));
    }
    for (int l = 0; l < 4; ++l) {                 // level 4 -> 1
        const int ci = cb >> l, co = ci / 2, S = 28 << l;
        const std::string d = "dec" + std::to_string(4 - l);
        T.up[l].t = t; T.up[l].cin = ci; T.up[l].cout = co;
        t += 2;
        T.dec[l][0] = conv(2 * co, 2 * co, co, S, false, d + "conv1", d + "norm1");
        T.dec[l][1] = conv(co, co, co, S, false, d + "conv2", d + "norm2");
    }
    T.head_t = t;
    T.n_tensors = t + 2;
    T.n_bn = bn;
}

int check_args(const SmkGenerator* h, const SmkGeneratorTrainArgs* a, const char* fn) {
    SMK_REQUIRE(h && h->train, "%s: not a train-mode handle (smk_generator_train_create)", fn);
    SMK_REQUIRE(a && a->tensors && a->num_batches_tracked, "%s: null args", fn);
    SMK_REQUIRE(a->n_tensors == h->topo.n_tensors, "%s: expects %d tensors (state_dict order, num_batches_tracked removed), got %d", fn,
                h->topo.n_tensors, a->n_tensors);
    for (int k = 0; k < a->n_tensors; ++k) SMK_REQUIRE(a->tensors[k], "%s: null tensor %d", fn, k);
    for (int k = 0; k < h->topo.n_bn; ++k) SMK_REQUIRE(a->num_batches_tracked[k], "%s: null num_batches_tracked %d", fn, k);
    SMK_REQUIRE(a->momentum <= 1.f && a->eps > 0.f, "%s: momentum must be in [0, 1] (or negative for None) and eps > 0", fn);
    return 0;
}

}  // namespace

extern "C" int smk_generator_train_create(int in_channels, int out_channels, int init_features, int res_blocks, int precision, SmkGenerator** out) {
    SMK_REQUIRE(out, "smk_generator_train_create: null argument");
    SMK_REQUIRE(precision == 0 || precision == 1 || precision == 3, "smk_generator_train_create: precision must be 0, 1 or 3");
    SMK_REQUIRE(init_features > 0 && init_features % 8 == 0 && out_channels >= 1 && out_channels <= 4 && in_channels >= 1 && res_blocks >= 0,
                "smk_generator_train_create: need init_features %% 8 == 0, out_channels in [1, 4], in_channels >= 1, res_blocks >= 0");
    SMK_REQUIRE(precision == 0 || init_features % 32 == 0, "smk_generator_train_create: the tensor-core path needs init_features %% 32 == 0");
    if (precision != 0) { if (int rc = smk::tc_init()) return rc; }
    SmkGenerator* h = new SmkGenerator();
    h->train = true;
    h->cin = in_channels; h->cout = out_channels; h->f = init_features; h->nres = res_blocks; h->precision = precision;
    h->cin_p = precision != 0 ? (in_channels + 31) & ~31 : (in_channels + 7) & ~7;
    build_topology(h);
    // unit scales / zero biases of every GEMM epilogue: N <= 4 * 8f (the first up-convolution) or cin_p
    const std::vector<float> one((size_t)std::max(32 * h->f, h->cin_p), 1.f), zero(one.size(), 0.f);
    cudaError_t e = h->arena.upload(one, &h->ones);
    if (e == cudaSuccess) e = h->arena.upload(zero, &h->zeros);
    if (e != cudaSuccess) { smk::set_error("smk_generator_train_create: %s", cudaGetErrorString(e)); delete h; return (int)e; }
    *out = h;
    return 0;
}

extern "C" size_t smk_generator_train_workspace_bytes(const SmkGenerator* h, int B) {
    return h && h->train && B > 0 ? ws_bytes(h, B) : 0;
}

extern "C" int smk_generator_forward_train(const SmkGenerator* h, const SmkGeneratorTrainArgs* args, const float* x, int B, float* y,
                                           float* saved, size_t saved_bytes, void* ws, size_t ws_bytes_, void* stream) {
    const char* fn = "smk_generator_forward_train";
    if (int rc = check_args(h, args, fn)) return rc;
    SMK_REQUIRE(B >= 0, "%s: negative batch", fn);
    if (B == 0) return 0;
    SMK_REQUIRE(x && y, "%s: null input or output", fn);
    const size_t sv_bytes = smk_generator_saved_bytes(h, B), need = smk_generator_train_workspace_bytes(h, B);
    SMK_REQUIRE(!saved || saved_bytes >= sv_bytes, "%s: saved buffer too small", fn);
    SMK_REQUIRE(ws && ws_bytes_ >= need + (saved ? 0 : sv_bytes), "%s: workspace too small (without `saved` it also holds the activations)", fn);
    cudaStream_t st = (cudaStream_t)stream;
    smk::Workspace w(ws, ws_bytes_);
    Ws W;
    SMK_REQUIRE(carve(w, h, B, &W), "%s: workspace carve-up failed", fn);
    float* sv = saved ? saved : w.take<float>(sv_bytes / 4);
    SMK_REQUIRE(sv, "%s: workspace carve-up failed", fn);
    const TrainTopo& T = h->topo;
    float* stats = sv + (size_t)B * h->saved.total;
    auto SV = [&](int k) { return sv + (size_t)B * h->saved.off[k]; };
    const bool tc = h->precision != 0, rnd = h->precision == 1;     // TF32: activations that feed a GEMM are rounded
    const float eps = args->eps, mom = args->momentum;
    const int f = h->f, cb = 16 * f;
    Packed P;
    int rc = pack_weights(h, args, false, W.pk, &P, st);
    if (rc) return rc;
    // conv + BatchNorm (+ res) (+ ReLU) of one layer into `out`
    auto layer = [&](const smk::GemmW& wt, const TrainConv& c, const float* in, int ld_in, const float* res, bool relu, bool round, const BnOut& out) {
        int r = conv3(h, wt, c, in, ld_in, B, SV(c.sv_z), st);
        if (r) return r;
        float* mean = stats + c.stats;
        return bn_forward(bn_ref(args, nullptr, c), SV(c.sv_z), (long)B * c.S * c.S, c.cout, eps, mom, mean, mean + c.cout, res, relu, round, out,
                          W.part, st);
    };
    if ((rc = smk::nchw_to_nhwc_pad(x, B, h->cin, 224, 224, h->cin_p, SV(T.sv_input), st, rnd))) return rc;
    // encoder levels: conv1; conv2 -> the skip half of the decoder's input; pool
    const float* in = SV(T.sv_input); int ld = h->cin_p;
    for (int l = 0; l < 4; ++l) {
        const int S = 224 >> l, c = f << l;
        const TrainConv &c1 = T.enc[l][0], &c2 = T.enc[l][1];
        if ((rc = layer(P.enc[2 * l], c1, in, ld, nullptr, true, rnd, BnOut{SV(c1.sv_y), c}))) return rc;
        float* skip = SV(T.sv_cat[l]) + c;
        if ((rc = layer(P.enc[2 * l + 1], c2, SV(c1.sv_y), c, nullptr, true, rnd, BnOut{skip, 2 * c}))) return rc;
        if ((rc = smk::maxpool2x2(skip, 2 * c, B, S, S, c, SV(T.sv_pool[l]), st))) return rc;
        in = SV(T.sv_pool[l]); ld = c;
    }
    // bottleneck and ResNet blocks; at precisions 1 and 3 every input of a reflection-padded conv is also written into a
    // padded buffer (xa: the residual stream, xt: the block's inner activation)
    float *xa = W.pad[0], *xt = W.pad[1];
    auto padded = [&](float* y, int ld_y, float* pad) { return BnOut{y, ld_y, tc ? pad : nullptr, B, 14, 14}; };
    const TrainConv &b1 = T.enc[4][0], &b2 = T.enc[4][1];
    if ((rc = layer(P.enc[8], b1, in, ld, nullptr, true, rnd, BnOut{SV(b1.sv_y), cb}))) return rc;
    if ((rc = layer(P.enc[9], b2, SV(b1.sv_y), cb, nullptr, true, rnd, padded(SV(b2.sv_y), cb, h->nres > 0 ? xa : nullptr)))) return rc;
    if (tc && h->nres > 0) { if ((rc = smk::reflect_halo(xa, B, 14, 14, cb, st))) return rc; }
    const float* xs = SV(b2.sv_y);                  // the residual stream, compact
    for (int r = 0; r < h->nres; ++r) {
        const TrainConv &r1 = T.res[2 * r], &r2 = T.res[2 * r + 1];
        const bool last = r == h->nres - 1;
        if ((rc = layer(P.res[2 * r], r1, tc ? xa : xs, cb, nullptr, true, rnd, padded(SV(r1.sv_y), cb, xt)))) return rc;
        if (tc) { if ((rc = smk::reflect_halo(xt, B, 14, 14, cb, st))) return rc; }
        if ((rc = layer(P.res[2 * r + 1], r2, tc ? xt : SV(r1.sv_y), cb, xs, false, rnd, padded(SV(r2.sv_y), cb, last ? nullptr : xa)))) return rc;
        if (tc && !last) { if ((rc = smk::reflect_halo(xa, B, 14, 14, cb, st))) return rc; }
        xs = SV(r2.sv_y);
    }
    // decoder levels 4..1: upconv -> the lower half of the decoder's input; conv1 over the concat; conv2
    const float* din = xs; int dS = 14;
    for (int l = 0; l < 4; ++l) {
        const int lvl = 3 - l;
        const TrainUp& u = T.up[l];
        smk::Conv q{};
        q.in = din; q.ld_in = u.cin; q.B = B; q.H = dS; q.W = dS; q.Cin = u.cin; q.wgt = P.up[l]; q.scale = h->ones; q.bias = P.up_bias[l];
        q.N = 4 * u.cout; q.K = u.cin; q.mode = 0; q.out = SV(T.sv_cat[lvl]); q.ld_out = 2 * u.cout; q.store = 1; q.round_out = rnd ? 1 : 0;
        if ((rc = smk::conv(q, st))) return rc;
        dS *= 2;
        const TrainConv &d1 = T.dec[l][0], &d2 = T.dec[l][1];
        if ((rc = layer(P.dec[2 * l], d1, SV(T.sv_cat[lvl]), 2 * u.cout, nullptr, true, rnd, BnOut{SV(d1.sv_y), u.cout}))) return rc;
        // the head's input (dec1norm2) feeds the fp32 1x1 conv: not rounded
        if ((rc = layer(P.dec[2 * l + 1], d2, SV(d1.sv_y), u.cout, nullptr, true, rnd && l < 3, BnOut{SV(d2.sv_y), u.cout}))) return rc;
        din = SV(d2.sv_y);
    }
    return smk::conv1x1_sigmoid_nchw(din, B, 224 * 224, f, P.head_w, args->tensors[T.head_t + 1], h->cout, y, st);
}

extern "C" int smk_generator_backward_train(const SmkGenerator* h, const SmkGeneratorTrainArgs* args, int B, const float* y, const float* saved,
                                            size_t saved_bytes, const float* g_y, float* g_x, const SmkGeneratorTrainGrads* grads, void* ws,
                                            size_t ws_bytes_, void* stream) {
    const char* fn = "smk_generator_backward_train";
    if (int rc = check_args(h, args, fn)) return rc;
    SMK_REQUIRE(B >= 0, "%s: negative batch", fn);
    if (B == 0) return 0;
    SMK_REQUIRE(y && saved && g_y, "%s: null output, saved buffer or output gradient", fn);
    SMK_REQUIRE(saved_bytes >= smk_generator_saved_bytes(h, B), "%s: saved buffer too small", fn);
    SMK_REQUIRE(ws && ws_bytes_ >= smk_generator_train_workspace_bytes(h, B), "%s: workspace too small", fn);
    const TrainTopo& T = h->topo;
    bool stats_grad = false;
    if (grads && grads->tensors) each_conv(T, [&](const TrainConv& c) { stats_grad = stats_grad || grads->tensors[c.t + 3] || grads->tensors[c.t + 4]; });
    SMK_REQUIRE(!stats_grad, "%s: running statistics have no gradient", fn);
    cudaStream_t st = (cudaStream_t)stream;
    smk::Workspace w(ws, ws_bytes_);
    Ws W;
    SMK_REQUIRE(carve(w, h, B, &W), "%s: workspace carve-up failed", fn);
    const float* stats = saved + (size_t)B * h->saved.total;
    auto SV = [&](int k) { return const_cast<float*>(saved) + (size_t)B * h->saved.off[k]; };
    const bool rnd = h->precision == 1;              // gradients that feed a TF32 GEMM are rounded
    const int f = h->f, cb = 16 * f;
    auto gt = [&](int t) -> float* { return grads && grads->tensors ? grads->tensors[t] : nullptr; };
    Packed P;
    int rc = pack_weights(h, args, true, W.pk, &P, st);
    if (rc) return rc;
    // BatchNorm backward of layer c (g -> gz, may alias; y: the ReLU mask, null for none) and its weight gradient over the
    // conv's input a (pixel stride lda, first c.cin channels)
    auto bn_wgrad = [&](const TrainConv& c, const float* g, const float* ymask, float* gz, const float* a, int lda) {
        const float* mean = stats + c.stats;
        const BnRef r = bn_ref(args, grads, c);
        int e = bn_backward(r, g, ymask, SV(c.sv_z), mean, mean + c.cout, (long)B * c.S * c.S, c.cout, rnd, gz, W.part, W.gb, st);
        if (e || !r.gw) return e;
        return conv3_wgrad(gz, a, lda, B, c.S, c.S, c.cin, c.cout, c.refl, W.wpart, r.gw, st);
    };
    // round: the result feeds a TF32 GEMM directly (not through a BatchNorm backward, which rounds its own output)
    auto dgrad = [&](const smk::GemmW& wt, const TrainConv& c, const float* g, int S, float* out, int ld_out, bool round = false) {
        return gen::dgrad3(wt, c.cin_p, c.cout, h->ones, h->zeros, g, B, S, nullptr, out, ld_out, round, st);
    };
    float *A = W.g[0], *Bf = W.g[1];
    // head: the sigmoid and the 1x1 conv (weight and bias gradients over the head's input), through dec1conv2's ReLU
    const float* d = SV(T.dec[3][1].sv_y);
    const long HW = 224 * 224;
    if (gt(T.head_t) || gt(T.head_t + 1)) {
        float* t = W.s2d;
        SMK_TAG("head_sigmoid_dgrad", 4.0 * B * HW * 3.0 * h->cout, 3.0 * B * HW * h->cout, st);
        SMK_LAUNCH(sigmoid_bwd_kernel, dim3(cdiv((long)B * HW * h->cout, 256)), dim3(256), 0, st, g_y, y, B, (int)HW, h->cout, t);
        SMK_CHECK_LAUNCH();
        if (gt(T.head_t)) { if ((rc = pw_wgrad(t, d, B * HW, h->cout, f, W.wpart, gt(T.head_t), st))) return rc; }
        if (gt(T.head_t + 1)) { if ((rc = channel_sum(t, B * HW, h->cout, gt(T.head_t + 1), W.part, W.gb, st))) return rc; }
    }
    if ((rc = gen::head_bwd(g_y, y, B, (int)HW, h->cout, P.head_w, d, f, rnd, A, st))) return rc;
    // decoder levels 1..4: conv2, conv1 (both halves of the concat), up-convolution
    for (int lvl = 0; lvl < 4; ++lvl) {
        const int i = 3 - lvl, S = 224 >> lvl, c = f << lvl;
        const TrainConv &d1 = T.dec[i][0], &d2 = T.dec[i][1];
        const TrainUp& u = T.up[i];
        if ((rc = bn_wgrad(d2, A, SV(d2.sv_y), A, SV(d1.sv_y), c))) return rc;
        if ((rc = dgrad(P.dec[2 * i + 1], d2, A, S, Bf, c))) return rc;
        if ((rc = bn_wgrad(d1, Bf, SV(d1.sv_y), Bf, SV(T.sv_cat[lvl]), 2 * c))) return rc;
        if ((rc = dgrad(P.dec[2 * i], d1, Bf, S, W.gcat[lvl], 2 * c, rnd))) return rc;     // its lower half feeds dgrad_up
        if ((rc = gen::s2d(W.gcat[lvl], 2 * c, B, S / 2, c, W.s2d, st))) return rc;
        const long Mu = (long)B * (S / 2) * (S / 2);
        const float* up_in = lvl < 3 ? SV(T.dec[i - 1][1].sv_y) : SV(h->nres > 0 ? T.res.back().sv_y : T.enc[4][1].sv_y);
        if (float* gw = gt(u.t)) {
            if ((rc = pw_wgrad(up_in, W.s2d, Mu, u.cin, 4 * u.cout, W.wpart, W.upw, st))) return rc;
            const long n = (long)u.cin * u.cout * 4;
            SMK_TAG("upconv_wgrad_order", 8.0 * n, 0.0, st);
            SMK_LAUNCH(upconv_wgrad_order_kernel, dim3(cdiv(n, 256)), dim3(256), 0, st, W.upw, u.cin, u.cout, gw);
            SMK_CHECK_LAUNCH();
        }
        if (float* gbias = gt(u.t + 1)) { if ((rc = channel_sum(W.s2d, 4 * Mu, u.cout, gbias, W.part, W.gb, st))) return rc; }
        if ((rc = gen::dgrad_up(P.up[i], u.cin, u.cout, h->ones, h->zeros, W.s2d, B, S / 2, nullptr, A, false, st))) return rc;
    }
    // ResNet blocks, last to first: A holds the gradient of the block's output.  Each reflection-padded conv's dgrad runs over
    // a zero-haloed 16 x 16 copy of its output gradient, and fold maps the padded-domain result back (as the eval backward).
    float *gP = W.pad[0], *gpad = W.pad[1], *gz = W.pad[2], *gu = W.pad[3];
    for (int r = h->nres - 1; r >= 0; --r) {
        const TrainConv &r1 = T.res[2 * r], &r2 = T.res[2 * r + 1];
        const float* x_in = SV(r > 0 ? T.res[2 * r - 1].sv_y : T.enc[4][1].sv_y);
        if ((rc = bn_wgrad(r2, A, nullptr, gz, SV(r1.sv_y), cb))) return rc;
        if ((rc = gen::fold(nullptr, gz, 0, nullptr, B, cb, rnd, gpad, 1, st))) return rc;
        if ((rc = dgrad(P.res[2 * r + 1], r2, gpad, 16, gP, cb))) return rc;
        if ((rc = gen::fold(gP, nullptr, 0, nullptr, B, cb, false, gu, 0, st))) return rc;
        if ((rc = bn_wgrad(r1, gu, SV(r1.sv_y), gu, x_in, cb))) return rc;
        if ((rc = gen::fold(nullptr, gu, 0, nullptr, B, cb, rnd, gpad, 1, st))) return rc;
        if ((rc = dgrad(P.res[2 * r], r1, gpad, 16, gP, cb))) return rc;
        if ((rc = gen::fold(gP, A, 0, nullptr, B, cb, false, Bf, 0, st))) return rc;
        std::swap(A, Bf);
    }
    // bottleneck, then encoder levels 4..1: pool (+ skip gradient), conv2, conv1
    const TrainConv &b1 = T.enc[4][0], &b2 = T.enc[4][1];
    if ((rc = bn_wgrad(b2, A, SV(b2.sv_y), A, SV(b1.sv_y), cb))) return rc;
    if ((rc = dgrad(P.enc[9], b2, A, 14, Bf, cb))) return rc;
    if ((rc = bn_wgrad(b1, Bf, SV(b1.sv_y), Bf, SV(T.sv_pool[3]), 8 * f))) return rc;
    if ((rc = dgrad(P.enc[8], b1, Bf, 14, A, 8 * f))) return rc;
    float *g = A, *o = Bf;
    for (int lvl = 3; lvl >= 0; --lvl) {
        const int S = 224 >> lvl, c = f << lvl;
        const TrainConv &e1 = T.enc[lvl][0], &e2 = T.enc[lvl][1];
        float* cat = SV(T.sv_cat[lvl]);
        // pool_bwd applies conv2's ReLU mask (the skip is its output), so its BatchNorm backward takes no mask
        if ((rc = gen::pool_bwd(cat + c, 2 * c, g, W.gcat[lvl] + c, 2 * c, B, S, c, false, o, st))) return rc;
        if ((rc = bn_wgrad(e2, o, nullptr, o, SV(e1.sv_y), c))) return rc;
        if ((rc = dgrad(P.enc[2 * lvl + 1], e2, o, S, g, c))) return rc;
        const float* a = lvl > 0 ? SV(T.sv_pool[lvl - 1]) : SV(T.sv_input);
        if ((rc = bn_wgrad(e1, g, SV(e1.sv_y), g, a, lvl > 0 ? c / 2 : h->cin_p))) return rc;
        if (lvl == 0 && !g_x) return 0;              // an input without a gradient: no dgrad of the first conv
        if ((rc = dgrad(P.enc[2 * lvl], e1, g, S, o, lvl > 0 ? c / 2 : h->cin_p))) return rc;
        std::swap(g, o);
    }
    return gen::nhwc_to_nchw(g, B, 224 * 224, h->cin_p, h->cin, g_x, st);
}

// ---- test entry point: the host helper of the train path's 3x3 weight gradient -----------------------------------------

extern "C" int smk_debug_train_conv3_wgrad(const float* g, const float* a, int lda, int B, int H, int W, int cin, int cout, int reflect, float* out,
                                           void* ws, size_t ws_bytes_, void* stream) {
    const char* fn = "smk_debug_train_conv3_wgrad";
    SMK_REQUIRE(g && a && out && ws, "%s: null argument", fn);
    SMK_REQUIRE(B > 0 && H > 1 && W > 1 && cin > 0 && cout > 0 && lda >= cin, "%s: need B > 0, H, W > 1, cin, cout > 0 and lda >= cin", fn);
    smk::Workspace w(ws, ws_bytes_);
    float* part = w.take<float>(kWgradPart);
    SMK_REQUIRE(part, "%s: workspace too small", fn);
    return conv3_wgrad(g, a, lda, B, H, W, cin, cout, reflect != 0, part, out, (cudaStream_t)stream);
}
