// SmirkGenerator forward (UNet + ResNet blocks), eval-mode BatchNorm folded into conv epilogues.
//
// Replaces SmirkGenerator.forward (reference src/smirk_generator.py:51-86), `_block` (:88-119) and
// ResnetBlock (:121-178).  NHWC fp32 activations.  No tensor is materialised for torch.cat (:66-75):
// each skip tensor and each transposed-conv output is written straight into its channel slice of the
// decoder's input buffer by the producing kernel's strided epilogue; ConvTranspose2d(k2,s2) (:30-44)
// is one GEMM with N = 4*Cout and a pixel-shuffle store.
//
// precision 0: every convolution runs on the fp32 CUDA-core implicit GEMM (nn_kernels.cu); reflection
//              padding (:147-171) is resolved in the A-operand loader.
// precision 1: every convolution runs on the TF32 wgmma implicit GEMM (gemm_tc.cu); the very first one (Cin = 6)
//              reads an input whose channels are zero-padded to 32 by the layout-conversion kernel (one 128-byte
//              SWIZZLE_128B row per pixel: the im2col TMA path as is; 2.3x faster than the fp32 CUDA-core kernel it
//              replaces even though 26 of the 32 K-columns per tap multiply zeros).  The ResNet blocks keep their activations in
//              reflection-padded [B,16,16,512] buffers: each conv's epilogue writes the interior, a
//              tiny kernel mirrors the 1-pixel halo, and the next conv's im2col TMA reads it with no
//              padding — the hardware cannot reflect, so the halo is made explicit once per layer.
// precision 3: precision 1's launches with 3xTF32 arithmetic (gemm_tc's X3 = 3 instantiations): every weight, forward and
//              dgrad, is packed as a TF32 head plus a TF32 tail, the kernels split the activations themselves, and nothing
//              is rounded to TF32 between layers — fp32-equivalent results on the tensor cores.
//
// Input gradient (frozen weights, eval BN): smk_generator_forward_saved runs the same launches with the post-ReLU outputs
// of every block conv and ResNet conv1 written to a caller-owned `saved` buffer (by redirecting the store, or by a second
// store of the same epilogue), and smk_generator_backward walks the network backwards.  Every dgrad is an ordinary
// convolution on the forward's GEMM kernels: a 3x3 conv's g_x = conv3x3(g, W') with W'[ci][8 - tap][co] = s[co] W[co][ci][tap]
// (the folded BN scale rides in W', packed at create time next to the forward weights), the ReLU mask [a > 0] is applied
// by the epilogue of the kernel that produces g, and ConvTranspose2d's dgrad is a GEMM over a space-to-depth copy of g.
#include "nn_kernels.cuh"
#include "gemm_tc.cuh"
#include "generator.cuh"
#include <math.h>
#include <algorithm>
#include <string>

namespace {

using smk::TensorCursor;
using smk::grid_of;
constexpr float kBnEps = 1e-5f;

bool fold_conv3(TensorCursor& cur, int cin, int cin_p, int cout, bool tc, bool x3, smk::DeviceArena& arena, Conv3* out, cudaError_t* err) {
    const float* w = cur.next(); const float* g = cur.next(); const float* b = cur.next();
    const float* mu = cur.next(); const float* var = cur.next();
    if (!w || !g || !b || !mu || !var) return false;
    std::vector<float> S(cout), Bi(cout);
    smk::fold_bn(g, b, mu, var, cout, kBnEps, S.data(), Bi.data());
    out->cin = cin; out->cin_p = cin_p; out->cout = cout;
    cudaError_t e = smk::pack_conv3(w, S.data(), cin, cin_p, cout, tc, x3, arena, &out->fwd, &out->dgrad);
    if (e == cudaSuccess) e = arena.upload(S, &out->scale);
    if (e == cudaSuccess) e = arena.upload(Bi, &out->bias);
    *err = e;
    return e == cudaSuccess;
}

bool fold_upconv(TensorCursor& cur, int cin, int cout, bool tc, bool x3, smk::DeviceArena& arena, UpConv* out, cudaError_t* err) {
    const float* w = cur.next(); const float* b = cur.next();        // weight [cin, cout, 2, 2], bias [cout]
    if (!w || !b) return false;
    const int N = 4 * cout;                                         // n = q * cout + o, q = dy*2+dx
    std::vector<float> S((size_t)N, 1.f), Bi((size_t)N);
    for (int q = 0; q < 4; ++q) for (int o = 0; o < cout; ++o) Bi[q * cout + o] = b[o];
    out->cin = cin; out->cout = cout;
    cudaError_t e = smk::pack_gemm(arena, N, cin, tc, x3, [&](int n, int c) { return w[((size_t)c * cout + n % cout) * 4 + n / cout]; }, &out->fwd);
    if (e == cudaSuccess) e = smk::pack_gemm(arena, cin, N, tc, x3, [&](int c, int k) { return w[((size_t)c * cout + k % cout) * 4 + k / cout]; }, &out->dgrad);
    if (e == cudaSuccess) e = arena.upload(S, &out->scale);
    if (e == cudaSuccess) e = arena.upload(Bi, &out->bias);
    *err = e;
    return e == cudaSuccess;
}

}  // namespace

extern "C" int smk_generator_create(const SmkGeneratorDesc* desc, SmkGenerator** out) {
    SMK_REQUIRE(desc && out && desc->tensors, "smk_generator_create: null argument");
    SMK_REQUIRE(desc->precision == 0 || desc->precision == 1 || desc->precision == 3,
                "smk_generator_create: precision must be 0, 1 or 3 (0 = fp32 CUDA cores, 1 = TF32 wgmma, 3 = 3xTF32 wgmma: fp32-equivalent)");
    SMK_REQUIRE(desc->init_features % 8 == 0 && desc->out_channels <= 4 && desc->in_channels >= 1,
                "smk_generator_create: need init_features %% 8 == 0 and out_channels <= 4");
    SMK_REQUIRE(desc->precision == 0 || desc->init_features % 32 == 0, "smk_generator_create: the tensor-core path needs init_features %% 32 == 0");
    const bool tc = desc->precision != 0, x3 = desc->precision == 3;     // tensor cores; 3xTF32 arithmetic on them
    if (tc) { if (int rc = smk::tc_init()) return rc; }
    SmkGenerator* h = new SmkGenerator();
    h->cin = desc->in_channels; h->cout = desc->out_channels;
    h->cin_p = tc ? (desc->in_channels + 31) & ~31 : (desc->in_channels + 7) & ~7;
    h->f = desc->init_features; h->nres = desc->res_blocks; h->precision = desc->precision;
    const int f = h->f;
    TensorCursor cur{desc->tensors, desc->n_tensors};
    cudaError_t e = cudaSuccess;
    bool ok = true;
    int c_in = h->cin, c_in_p = h->cin_p;
    for (int l = 0; ok && l < 5; ++l) {
        int co = f << l;
        ok = fold_conv3(cur, c_in, c_in_p, co, tc, x3, h->arena, &h->enc[l][0], &e) &&
             fold_conv3(cur, co, co, co, tc, x3, h->arena, &h->enc[l][1], &e);
        c_in = c_in_p = co;
    }
    h->res.resize((size_t)2 * h->nres);
    for (int r = 0; ok && r < 2 * h->nres; ++r) ok = fold_conv3(cur, 16 * f, 16 * f, 16 * f, tc, x3, h->arena, &h->res[r], &e);
    for (int l = 0; ok && l < 4; ++l) {          // level 4 -> 1
        int ci = (16 * f) >> l, co = ci / 2;
        ok = fold_upconv(cur, ci, co, tc, x3, h->arena, &h->up[l], &e) && fold_conv3(cur, 2 * co, 2 * co, co, tc, x3, h->arena, &h->dec[l][0], &e) &&
             fold_conv3(cur, co, co, co, tc, x3, h->arena, &h->dec[l][1], &e);
    }
    if (ok) {
        const float* w = cur.next(); const float* b = cur.next();
        ok = w && b;
        if (ok) {
            std::vector<float> W((size_t)f * h->cout);
            for (int o = 0; o < h->cout; ++o) for (int c = 0; c < f; ++c) W[(size_t)c * h->cout + o] = w[(size_t)o * f + c];
            e = h->arena.upload(W, &h->fw);
            if (e == cudaSuccess) e = h->arena.upload(b, (size_t)h->cout, &h->fb);
            const std::vector<float> one((size_t)std::max(16 * f, h->cin_p), 1.f), zero(one.size(), 0.f);
            if (e == cudaSuccess) e = h->arena.upload(one, &h->ones);
            if (e == cudaSuccess) e = h->arena.upload(zero, &h->zeros);
            ok = e == cudaSuccess;
        }
    }
    if (!ok || cur.i != cur.n) {
        if (e != cudaSuccess) smk::set_error("smk_generator_create: upload failed: %s", cudaGetErrorString(e));
        else smk::set_error("smk_generator_create: consumed %d tensors but %d were given (state_dict order, num_batches_tracked removed)", cur.i, cur.n);
        delete h; return e != cudaSuccess ? (int)e : -1;
    }
    // every size is a multiple of 64 floats (init_features % 8 == 0), so the tensors are packed with no gaps
    auto add = [h](const std::string& name, int S, int C) { h->saved.add(name, S, S, C); };
    for (int l = 0; l < 4; ++l)
        for (int j = 1; j <= 2; ++j) add("enc" + std::to_string(l + 1) + "conv" + std::to_string(j), 224 >> l, f << l);
    add("bottleneckconv1", 14, 16 * f); add("bottleneckconv2", 14, 16 * f);
    for (int r = 0; r < h->nres; ++r) add("res" + std::to_string(r) + "conv1", 14, 16 * f);
    for (int l = 3; l >= 0; --l)
        for (int j = 1; j <= 2; ++j) add("dec" + std::to_string(l + 1) + "conv" + std::to_string(j), 224 >> l, f << l);
    *out = h;
    return 0;
}

extern "C" void smk_generator_destroy(SmkGenerator* h) { delete h; }

namespace {
// floats per image for every activation buffer (224x224 input)
struct Plan {
    size_t x8, cat[4], t[4], d[4], p[4], tb, b0, b1, pad[3];
    size_t total() const {
        size_t s = x8 + tb + b0 + b1 + pad[0] + pad[1] + pad[2];
        for (int i = 0; i < 4; ++i) s += cat[i] + t[i] + d[i] + p[i];
        return s;
    }
};
Plan make_plan(const SmkGenerator* h) {
    Plan P{};
    const size_t S = 224;
    P.x8 = S * S * h->cin_p;
    for (int l = 0; l < 4; ++l) {
        size_t s = S >> l, c = (size_t)h->f << l;
        P.cat[l] = s * s * 2 * c; P.t[l] = s * s * c; P.d[l] = s * s * c; P.p[l] = (s / 2) * (s / 2) * c;
    }
    size_t sb = S >> 4, cb = (size_t)h->f * 16;
    P.tb = P.b0 = P.b1 = sb * sb * cb;
    P.pad[0] = P.pad[1] = P.pad[2] = h->precision != 0 ? (sb + 2) * (sb + 2) * cb : 0;
    return P;
}

// One 3x3 convolution, dispatched on the handle's precision.
//   refl   : reflection padding (ResNet blocks).  At precisions 1 and 3 `in` must then be a padded buffer.
//   store  : 0 plain / slice, 2 interior of a padded buffer (precisions 1 and 3 only)
//   out2   : optional second, compact [B,S,S,cout] store of the activations (the grad-mode forward's saved copy)
int conv3(const SmkGenerator* h, const Conv3& c, const float* in, int ld_in, int B, int S, bool refl, bool relu,
          const float* res, int res_pad, float* out, int ld_out, int store, cudaStream_t st, bool fuse_head = false,
          float* out2 = nullptr) {
    smk::Conv p{};
    if (fuse_head) { p.head_w = h->fw; p.head_b = h->fb; p.head_c = h->cout; }
    p.in = in; p.ld_in = ld_in; p.B = B; p.H = S; p.W = S; p.Cin = c.cin_p; p.wgt = c.fwd; p.scale = c.scale; p.bias = c.bias;
    p.N = c.cout; p.K = 9 * c.cin_p; p.mode = refl ? 2 : 1; p.relu = relu ? 1 : 0;
    p.res = res; p.ld_res = c.cout; p.res_pad = res_pad; p.out = out; p.ld_out = ld_out; p.store = store;
    p.round_out = c.fwd.wt && !c.fwd.wt_lo ? 1 : 0;    // TF32 consumers; 3xTF32 consumers split full fp32 activations themselves
    p.out2 = out2; p.ld_out2 = c.cout;
    return smk::conv(p, st);
}

// Index of a saved tensor (forward order, see smk_generator_create).
int sv_enc(int l, int j) { return 2 * l + j; }                              // encoder level l (0 = 224^2), conv j (0, 1)
int sv_bott(int j) { return 8 + j; }
int sv_res(int r) { return 10 + r; }
int sv_dec(const SmkGenerator* h, int lvl, int j) { return 10 + h->nres + 2 * (3 - lvl) + j; }

// The forward.  sv == null: the forward-only path.  Otherwise every saved activation is written to sv as well: the
// layers whose output feeds only the next layer write straight into sv, the others (the skips, the padded ResNet
// stream and the fused head's input) store it a second time from the same epilogue.  The arithmetic is the same.
int generator_forward(const SmkGenerator* h, const float* x, int B, float* y, float* sv, void* ws, size_t ws_bytes, cudaStream_t st) {
    smk::Workspace w(ws, ws_bytes);
    const Plan P = make_plan(h);
    const int f = h->f;
    const bool tc = h->precision != 0;             // tensor cores (TF32 or 3xTF32): padded ResNet stream, fused head
    auto SV = [&](int i) -> float* { return sv ? sv + (size_t)B * h->saved.off[i] : nullptr; };
    float* x8 = w.take<float>(P.x8 * B);
    float *cat[4], *t[4], *d[4], *p[4];
    for (int l = 0; l < 4; ++l) {
        cat[l] = w.take<float>(P.cat[l] * B); t[l] = w.take<float>(P.t[l] * B);
        d[l] = w.take<float>(P.d[l] * B); p[l] = w.take<float>(P.p[l] * B);
    }
    float* tb = w.take<float>(P.tb * B); float* b0 = w.take<float>(P.b0 * B); float* b1 = w.take<float>(P.b1 * B);
    float* pad[3] = {nullptr, nullptr, nullptr};
    if (tc) for (int i = 0; i < 3; ++i) pad[i] = w.take<float>(P.pad[i] * B);
    SMK_REQUIRE(b1 != nullptr && (!tc || pad[2] != nullptr), "smk_generator_forward: workspace carve-up failed");
    int rc = smk::nchw_to_nhwc_pad(x, B, h->cin, 224, 224, h->cin_p, x8, st, h->precision == 1);
    if (rc) return rc;
    // encoder levels: conv1 -> t[l]; conv2 -> upper half of cat[l] (the skip); pool -> p[l]
    const float* in = x8; int ld = h->cin_p;
    for (int l = 0; l < 4; ++l) {
        int S = 224 >> l, c = f << l;
        float* e1 = sv ? SV(sv_enc(l, 0)) : t[l];
        if ((rc = conv3(h, h->enc[l][0], in, ld, B, S, false, true, nullptr, 0, e1, c, 0, st))) return rc;
        if ((rc = conv3(h, h->enc[l][1], e1, c, B, S, false, true, nullptr, 0, cat[l] + c, 2 * c, 0, st, false, SV(sv_enc(l, 1))))) return rc;
        if ((rc = smk::maxpool2x2(cat[l] + c, 2 * c, B, S, S, c, p[l], st))) return rc;
        in = p[l]; ld = c;
    }
    const int Sb = 14, cb = 16 * f;
    float* tbo = sv ? SV(sv_bott(0)) : tb;
    if ((rc = conv3(h, h->enc[4][0], p[3], 8 * f, B, Sb, false, true, nullptr, 0, tbo, cb, 0, st))) return rc;
    const float* bott;                              // plain [B,14,14,cb] tensor feeding the first upconv
    if (!tc || h->nres == 0) {
        float* b0o = sv ? SV(sv_bott(1)) : b0;
        if ((rc = conv3(h, h->enc[4][1], tbo, cb, B, Sb, false, true, nullptr, 0, b0o, cb, 0, st))) return rc;
        float* cur = b0o;
        float* const nxt[2] = {b1, b0};
        for (int r = 0; r < h->nres && !tc; ++r) {  // x + BN(conv(reflpad(ReLU(BN(conv(reflpad(x)))))))
            float* u = sv ? SV(sv_res(r)) : tb;
            if ((rc = conv3(h, h->res[2 * r], cur, cb, B, Sb, true, true, nullptr, 0, u, cb, 0, st))) return rc;
            if ((rc = conv3(h, h->res[2 * r + 1], u, cb, B, Sb, true, false, cur, 0, nxt[r & 1], cb, 0, st))) return rc;
            cur = nxt[r & 1];
        }
        bott = cur;
    } else {
        // tensor-core path: residual stream lives in reflection-padded buffers  xa -> (xt) -> xb
        float *xa = pad[0], *xt = pad[1], *xb = pad[2];
        if ((rc = conv3(h, h->enc[4][1], tbo, cb, B, Sb, false, true, nullptr, 0, xa, cb, 2, st, false, SV(sv_bott(1))))) return rc;
        if ((rc = smk::reflect_halo(xa, B, Sb, Sb, cb, st))) return rc;
        for (int r = 0; r < h->nres; ++r) {
            const bool last = r == h->nres - 1;
            if ((rc = conv3(h, h->res[2 * r], xa, cb, B, Sb, true, true, nullptr, 0, xt, cb, 2, st, false, SV(sv_res(r))))) return rc;
            if ((rc = smk::reflect_halo(xt, B, Sb, Sb, cb, st))) return rc;
            if ((rc = conv3(h, h->res[2 * r + 1], xt, cb, B, Sb, true, false, xa, 1, last ? b0 : xb, cb, last ? 0 : 2, st))) return rc;
            if (!last) { if ((rc = smk::reflect_halo(xb, B, Sb, Sb, cb, st))) return rc; std::swap(xa, xb); }
        }
        bott = b0;
    }
    // decoder levels 4..1: upconv -> lower half of cat; conv1 over the concat; conv2
    const float* din = bott; int dS = Sb;
    for (int l = 0; l < 4; ++l) {
        int lvl = 3 - l;                            // index into cat/t/d (3 = 28x28 ... 0 = 224x224)
        const UpConv& u = h->up[l];
        smk::Conv q{};
        q.in = din; q.ld_in = u.cin; q.B = B; q.H = dS; q.W = dS; q.Cin = u.cin; q.wgt = u.fwd; q.scale = u.scale; q.bias = u.bias;
        q.N = 4 * u.cout; q.K = u.cin; q.mode = 0; q.out = cat[lvl]; q.ld_out = 2 * u.cout; q.store = 1; q.round_out = u.fwd.wt && !u.fwd.wt_lo ? 1 : 0;
        if ((rc = smk::conv(q, st))) return rc;
        dS *= 2;
        float* dt = sv ? SV(sv_dec(h, lvl, 0)) : t[lvl];
        if ((rc = conv3(h, h->dec[l][0], cat[lvl], 2 * u.cout, B, dS, false, true, nullptr, 0, dt, u.cout, 0, st))) return rc;
        // last layer of the tensor-core path: the 1x1 conv + sigmoid (smirk_generator.py:77-78,86) rides in the epilogue of
        // dec1conv2 — the [B,224,224,32] activation (6.4 MB per face) is neither written nor read back (the grad-mode forward
        // stores it once, for the backward's ReLU mask)
        const bool fuse_head = l == 3 && tc && u.cout <= 32;
        if (fuse_head) return conv3(h, h->dec[l][1], dt, u.cout, B, dS, false, true, nullptr, 0, y, u.cout, 3, st, true, SV(sv_dec(h, lvl, 1)));
        float* dd = sv ? SV(sv_dec(h, lvl, 1)) : d[lvl];
        if ((rc = conv3(h, h->dec[l][1], dt, u.cout, B, dS, false, true, nullptr, 0, dd, u.cout, 0, st))) return rc;
        din = dd;
    }
    return smk::conv1x1_sigmoid_nchw(din, B, 224 * 224, f, h->fw, h->fb, h->cout, y, st);
}

// ---- backward kernels ----------------------------------------------------------------------------------------------
// Head: g_d[b,p,c] = (sum_j W_h[c][j] * g_y[b,j,p] * y (1 - y)) * [d > 0], NCHW g_y / y -> NHWC [B,HW,f].
__global__ void __launch_bounds__(256)
head_bwd_kernel(const float* __restrict__ gy, const float* __restrict__ y, int B, int HW, int cout, const float* __restrict__ w,
                const float* __restrict__ d, int f, int round, float* __restrict__ out) {
    const int F4 = f >> 2;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * HW * F4) return;
    const int q = (int)(i % F4); const long pix = i / F4;
    const int b = (int)(pix / HW), r = (int)(pix - (long)b * HW);
    float t[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        t[j] = 0.f;
        if (j < cout) { const size_t o = ((size_t)b * cout + j) * HW + r; const float yv = __ldg(y + o); t[j] = __ldg(gy + o) * (yv * (1.f - yv)); }
    }
    const float4 m = __ldg(reinterpret_cast<const float4*>(d + (size_t)pix * f) + q);
    const float mk[4] = {m.x, m.y, m.z, m.w};
    float o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int c = 4 * q + e;
        float acc = 0.f;
        for (int j = 0; j < cout; ++j) acc = fmaf(__ldg(w + (size_t)c * cout + j), t[j], acc);
        acc = mk[e] > 0.f ? acc : 0.f;
        o[e] = round ? smk::round_tf32(acc) : acc;
    }
    reinterpret_cast<float4*>(out + (size_t)pix * f)[q] = make_float4(o[0], o[1], o[2], o[3]);
}

// MaxPool 2x2 backward + skip gradient + ReLU mask of the pool input e (= the encoder's conv2 output = the skip):
// g_e = (g_skip + [first maximum of the window, row-major] * g_p) * [e > 0].
__global__ void __launch_bounds__(256)
pool_bwd_kernel(const float* __restrict__ e, int ld_e, const float* __restrict__ gp, const float* __restrict__ gskip, int ld_skip,
                int B, int S, int C, int round, float* __restrict__ out) {
    const int Ho = S >> 1, C4 = C >> 2;
    const long total = (long)B * Ho * Ho * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4); const long pix = i / C4;
        const int ow = (int)(pix % Ho); const long t = pix / Ho; const int oh = (int)(t % Ho); const int b = (int)(t / Ho);
        const size_t p00 = ((size_t)b * S + 2 * oh) * S + 2 * ow;
        const size_t px[4] = {p00, p00 + 1, p00 + S, p00 + S + 1};
        float v[4][4], g[4][4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(e + px[k] * ld_e) + c4);
            const float4 s = __ldg(reinterpret_cast<const float4*>(gskip + px[k] * ld_skip) + c4);
            v[k][0] = a.x; v[k][1] = a.y; v[k][2] = a.z; v[k][3] = a.w;
            g[k][0] = s.x; g[k][1] = s.y; g[k][2] = s.z; g[k][3] = s.w;
        }
        const float4 gq = __ldg(reinterpret_cast<const float4*>(gp + (size_t)pix * C) + c4);
        const float gv[4] = {gq.x, gq.y, gq.z, gq.w};
#pragma unroll
        for (int ch = 0; ch < 4; ++ch) {
            const float mx = fmaxf(fmaxf(v[0][ch], v[1][ch]), fmaxf(v[2][ch], v[3][ch]));
            const int arg = v[0][ch] == mx ? 0 : v[1][ch] == mx ? 1 : v[2][ch] == mx ? 2 : 3;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float r = k == arg ? g[k][ch] + gv[ch] : g[k][ch];
                r = v[k][ch] > 0.f ? r : 0.f;
                g[k][ch] = round ? smk::round_tf32(r) : r;
            }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
            reinterpret_cast<float4*>(out + px[k] * C)[c4] = make_float4(g[k][0], g[k][1], g[k][2], g[k][3]);
    }
}

// Space-to-depth of the up-convolution's output gradient: out[b,h,w,(dy*2+dx)*C + c] = in[b,2h+dy,2w+dx,c] (S = out size).
__global__ void __launch_bounds__(256)
s2d_kernel(const float* __restrict__ in, int ld_in, int B, int S, int C, float* __restrict__ out) {
    const int C4 = C >> 2;
    const long total = (long)B * S * S * 4 * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4); long t = i / C4; const int q = (int)(t % 4); const long pix = t / 4;
        const int w = (int)(pix % S); t = pix / S; const int h = (int)(t % S); const int b = (int)(t / S);
        const size_t src = ((size_t)b * 2 * S + 2 * h + (q >> 1)) * 2 * S + 2 * w + (q & 1);
        reinterpret_cast<float4*>(out + (size_t)pix * 4 * C + (size_t)q * C)[c4] = __ldg(reinterpret_cast<const float4*>(in + src * ld_in) + c4);
    }
}

// Adjoint of ReflectionPad2d(1) (the transpose of reflect_halo): g[h,w] = sum of gP over the padded pixels that mirror
// onto (h,w), fixed order; + res (plain or the interior of a padded buffer); * [mask > 0].  gP may be null (g = res).
// out_pad: write [B,H+2,W+2,C] with a zero halo (the next dgrad's zero padding over the padded domain), else [B,H,W,C].
__global__ void __launch_bounds__(256)
fold_kernel(const float* __restrict__ gP, const float* __restrict__ res, int res_pad, const float* __restrict__ mask,
            int B, int H, int W, int C, int round, float* __restrict__ out, int out_pad) {
    const int C4 = C >> 2, Ho = H + 2 * out_pad, Wo = W + 2 * out_pad, Hp = H + 2, Wp = W + 2;
    const long total = (long)B * Ho * Wo * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4); const long pix = i / C4;
        const int ow = (int)(pix % Wo); const long t = pix / Wo; const int oh = (int)(t % Ho); const int b = (int)(t / Ho);
        const int h = oh - out_pad, w = ow - out_pad;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (h >= 0 && h < H && w >= 0 && w < W) {
            if (gP) {
                const int rows[2] = {h + 1, h == 1 ? 0 : (h == H - 2 ? H + 1 : -1)};
                const int cols[2] = {w + 1, w == 1 ? 0 : (w == W - 2 ? W + 1 : -1)};
#pragma unroll
                for (int a = 0; a < 2; ++a)
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        if (rows[a] < 0 || cols[c] < 0) continue;
                        const float4 v = __ldg(reinterpret_cast<const float4*>(gP + (((size_t)b * Hp + rows[a]) * Wp + cols[c]) * C) + c4);
                        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                    }
            }
            if (res) {
                const size_t rp = res_pad ? ((size_t)b * Hp + h + 1) * Wp + w + 1 : ((size_t)b * H + h) * W + w;
                const float4 v = __ldg(reinterpret_cast<const float4*>(res + rp * C) + c4);
                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
            if (mask) {
                const float4 m = __ldg(reinterpret_cast<const float4*>(mask + (((size_t)b * H + h) * W + w) * C) + c4);
                acc.x = m.x > 0.f ? acc.x : 0.f; acc.y = m.y > 0.f ? acc.y : 0.f; acc.z = m.z > 0.f ? acc.z : 0.f; acc.w = m.w > 0.f ? acc.w : 0.f;
            }
            if (round) { acc.x = smk::round_tf32(acc.x); acc.y = smk::round_tf32(acc.y); acc.z = smk::round_tf32(acc.z); acc.w = smk::round_tf32(acc.w); }
        }
        reinterpret_cast<float4*>(out + (size_t)pix * C)[c4] = acc;
    }
}

// First C of Cp channels, NHWC [B,HW,Cp] -> NCHW [B,C,HW].
__global__ void __launch_bounds__(256)
nhwc_to_nchw_kernel(const float* __restrict__ in, int B, int HW, int Cp, int C, float* __restrict__ out) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)B * C * HW) return;
    const int r = (int)(i % HW); const long t = i / HW; const int c = (int)(t % C); const int b = (int)(t / C);
    out[i] = __ldg(in + ((size_t)b * HW + r) * Cp + c);
}

// The eval handle's dgrads: its packed dgrad weights, which carry the folded BN scale.
int dgrad3(const SmkGenerator* h, const Conv3& c, const float* g, int B, int S, const float* mask, float* out, int ld_out, bool round,
           cudaStream_t st) {
    return gen::dgrad3(c.dgrad, c.cin_p, c.cout, h->ones, h->zeros, g, B, S, mask, out, ld_out, round, st);
}
int dgrad_up(const SmkGenerator* h, const UpConv& u, const float* s2d, int B, int S, const float* mask, float* out, bool round, cudaStream_t st) {
    return gen::dgrad_up(u.dgrad, u.cin, u.cout, h->ones, h->zeros, s2d, B, S, mask, out, round, st);
}
using gen::fold;

// floats per image of the backward's workspace buffers
struct GradPlan {
    size_t g, gcat[4], s2d, pad;
    size_t total() const { return 2 * g + gcat[0] + gcat[1] + gcat[2] + gcat[3] + s2d + 4 * pad; }
};
GradPlan make_grad_plan(const SmkGenerator* h) {
    GradPlan P{};
    P.g = (size_t)224 * 224 * std::max(h->f, h->cin_p);
    for (int l = 0; l < 4; ++l) { const size_t S = 224 >> l; P.gcat[l] = S * S * 2 * ((size_t)h->f << l); }
    P.s2d = (size_t)112 * 112 * 4 * h->f;
    P.pad = h->nres > 0 ? (size_t)16 * 16 * 16 * h->f : 0;
    return P;
}
}  // namespace

namespace gen {

int dgrad3(const smk::GemmW& w, int cin_p, int cout, const float* ones, const float* zeros, const float* g, int B, int S, const float* mask,
           float* out, int ld_out, bool round, cudaStream_t st) {
    smk::Conv p{};
    p.in = g; p.ld_in = cout; p.B = B; p.H = S; p.W = S; p.Cin = cout; p.wgt = w;
    p.scale = ones; p.bias = zeros;
    p.N = cin_p; p.K = 9 * cout; p.mode = 1; p.out = out; p.ld_out = ld_out; p.round_out = round ? 1 : 0;
    p.mask = mask; p.ld_mask = cin_p; p.tag = w.wt_lo ? "conv3x3_dgrad_tc3x" : w.wt ? "conv3x3_dgrad_tc" : "conv3x3_dgrad_f32";
    return smk::conv(p, st);
}

int dgrad_up(const smk::GemmW& w, int cin, int cout, const float* ones, const float* zeros, const float* s2d, int B, int S, const float* mask,
             float* out, bool round, cudaStream_t st) {
    const int K = 4 * cout;
    smk::Conv p{};
    p.in = s2d; p.ld_in = K; p.B = B; p.H = S; p.W = S; p.Cin = K; p.wgt = w;
    p.scale = ones; p.bias = zeros;
    p.N = cin; p.K = K; p.mode = 0; p.out = out; p.ld_out = cin; p.round_out = round ? 1 : 0;
    p.mask = mask; p.ld_mask = cin; p.tag = w.wt_lo ? "upconv_dgrad_tc3x" : w.wt ? "upconv_dgrad_tc" : "upconv_dgrad_f32";
    return smk::conv(p, st);
}

int s2d(const float* in, int ld_in, int B, int S, int C, float* out, cudaStream_t st) {
    const long total = (long)B * S * S * 4 * (C / 4);
    SMK_TAG("upconv_s2d", 32.0 * B * S * S * C, 0.0, st);
    SMK_LAUNCH(s2d_kernel, dim3(grid_of(total)), dim3(256), 0, st, in, ld_in, B, S, C, out);
    SMK_CHECK_LAUNCH();
    return 0;
}

int fold(const float* gP, const float* res, int res_pad, const float* mask, int B, int C, bool round, float* out, int out_pad, cudaStream_t st) {
    const int H = 14, Ho = H + 2 * out_pad;
    const long total = (long)B * Ho * Ho * (C / 4);
    SMK_TAG("reflect_fold", 4.0 * B * C * ((gP ? 16.0 * 16 : 0.0) + (res ? 196.0 : 0.0) + (mask ? 196.0 : 0.0) + Ho * Ho), (gP ? 1.0 : 0.0) * B * C * 256, st);
    SMK_LAUNCH(fold_kernel, dim3(grid_of(total)), dim3(256), 0, st, gP, res, res_pad, mask, B, H, H, C, round ? 1 : 0, out, out_pad);
    SMK_CHECK_LAUNCH();
    return 0;
}

int pool_bwd(const float* e, int ld_e, const float* gp, const float* gskip, int ld_skip, int B, int S, int C, bool round, float* out, cudaStream_t st) {
    const long total = (long)B * (S / 2) * (S / 2) * (C / 4);
    SMK_TAG("maxpool_dgrad", 4.0 * B * ((double)S * S * C * 3 + (S / 2.0) * (S / 2.0) * C), 0.0, st);
    SMK_LAUNCH(pool_bwd_kernel, dim3(grid_of(total)), dim3(256), 0, st, e, ld_e, gp, gskip, ld_skip, B, S, C, round ? 1 : 0, out);
    SMK_CHECK_LAUNCH();
    return 0;
}

int head_bwd(const float* gy, const float* y, int B, int HW, int cout, const float* w, const float* d, int f, bool round, float* out, cudaStream_t st) {
    const long total = (long)B * HW * (f / 4);
    SMK_TAG("head_dgrad", 4.0 * B * HW * (2.0 * cout + 2.0 * f), 2.0 * B * HW * f * cout, st);
    SMK_LAUNCH(head_bwd_kernel, dim3(smk::cdiv(total, 256)), dim3(256), 0, st, gy, y, B, HW, cout, w, d, f, round ? 1 : 0, out);
    SMK_CHECK_LAUNCH();
    return 0;
}

int nhwc_to_nchw(const float* in, int B, int HW, int Cp, int C, float* out, cudaStream_t st) {
    const long total = (long)B * C * HW;
    SMK_TAG("nhwc_to_nchw", 4.0 * (double)B * HW * (C + Cp), 0.0, st);
    SMK_LAUNCH(nhwc_to_nchw_kernel, dim3(smk::cdiv(total, 256)), dim3(256), 0, st, in, B, HW, Cp, C, out);
    SMK_CHECK_LAUNCH();
    return 0;
}

}  // namespace gen

extern "C" size_t smk_generator_workspace_bytes(const SmkGenerator* h, int B) {
    return (make_plan(h).total() * (size_t)B * sizeof(float)) + 40 * 256;
}

extern "C" int smk_generator_forward(const SmkGenerator* h, const float* x, int B, float* y,
                                     void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;                      // empty batch: nothing to do (pointers may be null)
    SMK_REQUIRE(h && x && y, "smk_generator_forward: null argument");
    SMK_REQUIRE(B > 0, "smk_generator_forward: negative batch");
    SMK_REQUIRE(ws && ws_bytes >= smk_generator_workspace_bytes(h, B), "smk_generator_forward: workspace too small");
    SMK_REQUIRE(!h->train, "smk_generator_forward: a train handle has no packed weights (smk_generator_forward_train)");
    return generator_forward(h, x, B, y, nullptr, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" size_t smk_generator_saved_bytes(const SmkGenerator* h, int B) {
    return h ? h->saved.bytes(B) + smk::ws_round(h->topo.stats_floats * sizeof(float)) : 0;     // stats: train handles only
}

extern "C" int smk_generator_saved_tensor(const SmkGenerator* h, int B, int i, const char** name, size_t* offset, int* dims) {
    return smk::saved_tensor(h ? &h->saved : nullptr, "smk_generator_saved_tensor", B, i, name, offset, dims);
}

extern "C" int smk_generator_forward_saved(const SmkGenerator* h, const float* x, int B, float* y, float* saved, size_t saved_bytes,
                                           void* ws, size_t ws_bytes, void* stream) {
    SMK_REQUIRE(h, "smk_generator_forward_saved: null handle");
    SMK_REQUIRE(B >= 0, "smk_generator_forward_saved: negative batch");
    if (B == 0) return 0;
    SMK_REQUIRE(x && y && saved, "smk_generator_forward_saved: null argument");
    SMK_REQUIRE(saved_bytes > 0 && saved_bytes >= smk_generator_saved_bytes(h, B), "smk_generator_forward_saved: saved buffer too small");
    SMK_REQUIRE(ws && ws_bytes > 0 && ws_bytes >= smk_generator_workspace_bytes(h, B), "smk_generator_forward_saved: workspace too small");
    SMK_REQUIRE(!h->train, "smk_generator_forward_saved: a train handle has no packed weights (smk_generator_forward_train)");
    return generator_forward(h, x, B, y, saved, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" size_t smk_generator_backward_workspace_bytes(const SmkGenerator* h, int B) {
    return h && B > 0 ? make_grad_plan(h).total() * (size_t)B * sizeof(float) + 16 * 256 : 0;
}

extern "C" int smk_generator_backward(const SmkGenerator* h, int B, const float* y, const float* saved, size_t saved_bytes,
                                      const float* g_y, float* g_x, void* ws, size_t ws_bytes, void* stream) {
    SMK_REQUIRE(h, "smk_generator_backward: null handle");
    SMK_REQUIRE(B >= 0, "smk_generator_backward: negative batch");
    if (B == 0) return 0;
    SMK_REQUIRE(y && saved && g_y && g_x, "smk_generator_backward: null argument");
    SMK_REQUIRE(saved_bytes > 0 && saved_bytes >= smk_generator_saved_bytes(h, B), "smk_generator_backward: saved buffer too small");
    SMK_REQUIRE(ws && ws_bytes > 0 && ws_bytes >= smk_generator_backward_workspace_bytes(h, B), "smk_generator_backward: workspace too small");
    SMK_REQUIRE(!h->train, "smk_generator_backward: a train handle (smk_generator_backward_train)");
    cudaStream_t st = (cudaStream_t)stream;
    const int f = h->f, cb = 16 * f;
    const bool rnd = h->precision == 1;            // TF32 rounding of every gradient a TF32 dgrad reads (not at 3xTF32)
    auto SV = [&](int i) -> const float* { return saved + (size_t)B * h->saved.off[i]; };
    const GradPlan P = make_grad_plan(h);
    smk::Workspace w(ws, ws_bytes);
    float* A = w.take<float>(P.g * B); float* Bf = w.take<float>(P.g * B);
    float* gcat[4];
    for (int l = 0; l < 4; ++l) gcat[l] = w.take<float>(P.gcat[l] * B);
    float* s2d = w.take<float>(P.s2d * B);
    float* pad[4] = {nullptr, nullptr, nullptr, nullptr};
    if (h->nres > 0) for (int i = 0; i < 4; ++i) pad[i] = w.take<float>(P.pad * B);
    SMK_REQUIRE(s2d && (h->nres == 0 || pad[3]), "smk_generator_backward: workspace carve-up failed");
    int rc;
    // head: sigmoid and the 1x1 conv, through dec1conv2's ReLU
    if ((rc = gen::head_bwd(g_y, y, B, 224 * 224, h->cout, h->fw, SV(sv_dec(h, 0, 1)), f, rnd, A, st))) return rc;
    // decoder levels 1..4: conv2, conv1 (both halves of the concat), up-convolution
    for (int lvl = 0; lvl < 4; ++lvl) {
        const int i = 3 - lvl, S = 224 >> lvl, c = f << lvl;
        if ((rc = dgrad3(h, h->dec[i][1], A, B, S, SV(sv_dec(h, lvl, 0)), Bf, c, rnd, st))) return rc;
        if ((rc = dgrad3(h, h->dec[i][0], Bf, B, S, nullptr, gcat[lvl], 2 * c, rnd, st))) return rc;
        if ((rc = gen::s2d(gcat[lvl], 2 * c, B, S / 2, c, s2d, st))) return rc;
        const float* m = lvl < 3 ? SV(sv_dec(h, lvl + 1, 1)) : (h->nres == 0 ? SV(sv_bott(1)) : nullptr);
        if ((rc = dgrad_up(h, h->up[i], s2d, B, S / 2, m, A, rnd, st))) return rc;
    }
    // ResNet blocks, last to first, over zero-haloed 16 x 16 gradient buffers: g_x = fold(conv(G(fold(conv(G(g)) * [u > 0])))) + g
    float* g = A;                                    // gradient of the bottleneck's conv2 output, [B,14,14,cb]
    if (h->nres > 0) {
        float *cur = pad[0], *nxt = pad[1], *gP = pad[2], *gu = pad[3];
        if ((rc = fold(nullptr, A, 0, nullptr, B, cb, rnd, cur, 1, st))) return rc;
        for (int r = h->nres - 1; r >= 0; --r) {
            if ((rc = dgrad3(h, h->res[2 * r + 1], cur, B, 16, nullptr, gP, cb, rnd, st))) return rc;
            if ((rc = fold(gP, nullptr, 0, SV(sv_res(r)), B, cb, rnd, gu, 1, st))) return rc;
            if ((rc = dgrad3(h, h->res[2 * r], gu, B, 16, nullptr, gP, cb, rnd, st))) return rc;
            if (r == 0) { if ((rc = fold(gP, cur, 1, SV(sv_bott(1)), B, cb, rnd, Bf, 0, st))) return rc; }
            else { if ((rc = fold(gP, cur, 1, nullptr, B, cb, rnd, nxt, 1, st))) return rc; std::swap(cur, nxt); }
        }
        g = Bf;
    }
    float* o = g == A ? Bf : A;
    if ((rc = dgrad3(h, h->enc[4][1], g, B, 14, SV(sv_bott(0)), o, cb, rnd, st))) return rc;
    if ((rc = dgrad3(h, h->enc[4][0], o, B, 14, nullptr, g, 8 * f, rnd, st))) return rc;
    // encoder levels 4..1: pool (+ skip gradient), conv2, conv1
    for (int lvl = 3; lvl >= 0; --lvl) {
        const int S = 224 >> lvl, c = f << lvl;
        if ((rc = gen::pool_bwd(SV(sv_enc(lvl, 1)), c, g, gcat[lvl] + c, 2 * c, B, S, c, rnd, o, st))) return rc;
        if ((rc = dgrad3(h, h->enc[lvl][1], o, B, S, SV(sv_enc(lvl, 0)), g, c, rnd, st))) return rc;
        const int n_in = lvl > 0 ? c / 2 : h->cin_p;
        if ((rc = dgrad3(h, h->enc[lvl][0], g, B, S, nullptr, o, n_in, rnd && lvl > 0, st))) return rc;
        std::swap(g, o);
    }
    return gen::nhwc_to_nchw(g, B, 224 * 224, h->cin_p, h->cin, g_x, st);
}
