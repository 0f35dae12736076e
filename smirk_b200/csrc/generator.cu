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
#include "nn_kernels.cuh"
#include "gemm_tc.cuh"
#include <math.h>

namespace {

using smk::ConvProblem;
using smk::TcConv;
constexpr float kBnEps = 1e-5f;

struct Conv3 { float* w; float* wt; float* scale; float* bias; int cin, cin_p, cout; };  // w: [9*cin_p][cout]; wt: [cout][9*cin_p]
struct UpConv { float* w; float* wt; float* scale; float* bias; int cin, cout; };         // w: [cin][4*cout];   wt: [4*cout][cin]

struct TensorCursor {
    const float* const* t; int n; int i = 0;
    const float* next() { return i < n ? t[i++] : nullptr; }
};

bool fold_conv3(TensorCursor& cur, int cin, int cin_p, int cout, bool tc, smk::DeviceArena& arena, Conv3* out, cudaError_t* err) {
    const float* w = cur.next(); const float* g = cur.next(); const float* b = cur.next();
    const float* mu = cur.next(); const float* var = cur.next();
    if (!w || !g || !b || !mu || !var) return false;
    const size_t K = (size_t)9 * cin_p;
    std::vector<float> W(K * cout, 0.f), S(cout), Bi(cout);
    for (int o = 0; o < cout; ++o)
        for (int c = 0; c < cin; ++c)
            for (int k = 0; k < 9; ++k) {
                float v = w[((size_t)o * cin + c) * 9 + k];
                if (tc) W[(size_t)o * K + (size_t)k * cin_p + c] = smk::round_tf32_host(v);   // [N][K], TF32-rounded
                else W[((size_t)k * cin_p + c) * cout + o] = v;                // [K][N]
            }
    for (int o = 0; o < cout; ++o) {
        float s = g[o] / sqrtf(var[o] + kBnEps);
        S[o] = s; Bi[o] = b[o] - mu[o] * s;
    }
    out->cin = cin; out->cin_p = cin_p; out->cout = cout; out->w = out->wt = nullptr;
    cudaError_t e = arena.upload(W, tc ? &out->wt : &out->w);
    if (e == cudaSuccess) e = arena.upload(S, &out->scale);
    if (e == cudaSuccess) e = arena.upload(Bi, &out->bias);
    *err = e;
    return e == cudaSuccess;
}

bool fold_upconv(TensorCursor& cur, int cin, int cout, bool tc, smk::DeviceArena& arena, UpConv* out, cudaError_t* err) {
    const float* w = cur.next(); const float* b = cur.next();        // weight [cin, cout, 2, 2], bias [cout]
    if (!w || !b) return false;
    std::vector<float> W((size_t)cin * 4 * cout), S((size_t)4 * cout, 1.f), Bi((size_t)4 * cout);
    for (int c = 0; c < cin; ++c)
        for (int o = 0; o < cout; ++o)
            for (int q = 0; q < 4; ++q) {
                float v = w[((size_t)c * cout + o) * 4 + q];
                if (tc) W[((size_t)q * cout + o) * cin + c] = smk::round_tf32_host(v);   // [N = 4*cout][K = cin]
                else W[(size_t)c * 4 * cout + q * cout + o] = v;               // [K][N]
            }
    for (int q = 0; q < 4; ++q) for (int o = 0; o < cout; ++o) Bi[q * cout + o] = b[o];
    out->cin = cin; out->cout = cout; out->w = out->wt = nullptr;
    cudaError_t e = arena.upload(W, tc ? &out->wt : &out->w);
    if (e == cudaSuccess) e = arena.upload(S, &out->scale);
    if (e == cudaSuccess) e = arena.upload(Bi, &out->bias);
    *err = e;
    return e == cudaSuccess;
}

}  // namespace

struct SmkGenerator {
    int cin, cin_p, cout, f, nres, precision;
    Conv3 enc[5][2];                 // encoder1..4, bottleneck
    std::vector<Conv3> res;          // 2 per ResnetBlock
    UpConv up[4];                    // upconv4..1  (index 0 = level 4)
    Conv3 dec[4][2];                 // decoder4..1
    float *fw = nullptr, *fb = nullptr;   // final 1x1: W[f][cout], bias
    smk::DeviceArena arena;
};

extern "C" int smk_generator_create(const SmkGeneratorDesc* desc, SmkGenerator** out) {
    SMK_REQUIRE(desc && out && desc->tensors, "smk_generator_create: null argument");
    SMK_REQUIRE(desc->precision == 0 || desc->precision == 1, "smk_generator_create: precision must be 0 (fp32) or 1 (tf32 wgmma)");
    SMK_REQUIRE(desc->init_features % 8 == 0 && desc->out_channels <= 4 && desc->in_channels >= 1,
                "smk_generator_create: need init_features %% 8 == 0 and out_channels <= 4");
    SMK_REQUIRE(desc->precision == 0 || desc->init_features % 32 == 0, "smk_generator_create: the tensor-core path needs init_features %% 32 == 0");
    if (desc->precision == 1) { if (int rc = smk::tc_init()) return rc; }
    SmkGenerator* h = new SmkGenerator();
    h->cin = desc->in_channels; h->cout = desc->out_channels;
    h->cin_p = desc->precision == 1 ? (desc->in_channels + 31) & ~31 : (desc->in_channels + 7) & ~7;
    h->f = desc->init_features; h->nres = desc->res_blocks; h->precision = desc->precision;
    const int f = h->f;
    const bool tc = h->precision == 1;
    TensorCursor cur{desc->tensors, desc->n_tensors};
    cudaError_t e = cudaSuccess;
    bool ok = true;
    int c_in = h->cin, c_in_p = h->cin_p;
    for (int l = 0; ok && l < 5; ++l) {
        int co = f << l;
        ok = fold_conv3(cur, c_in, c_in_p, co, tc, h->arena, &h->enc[l][0], &e) &&
             fold_conv3(cur, co, co, co, tc, h->arena, &h->enc[l][1], &e);
        c_in = c_in_p = co;
    }
    h->res.resize((size_t)2 * h->nres);
    for (int r = 0; ok && r < 2 * h->nres; ++r) ok = fold_conv3(cur, 16 * f, 16 * f, 16 * f, tc, h->arena, &h->res[r], &e);
    for (int l = 0; ok && l < 4; ++l) {          // level 4 -> 1
        int ci = (16 * f) >> l, co = ci / 2;
        ok = fold_upconv(cur, ci, co, tc, h->arena, &h->up[l], &e) && fold_conv3(cur, 2 * co, 2 * co, co, tc, h->arena, &h->dec[l][0], &e) &&
             fold_conv3(cur, co, co, co, tc, h->arena, &h->dec[l][1], &e);
    }
    if (ok) {
        const float* w = cur.next(); const float* b = cur.next();
        ok = w && b;
        if (ok) {
            std::vector<float> W((size_t)f * h->cout);
            for (int o = 0; o < h->cout; ++o) for (int c = 0; c < f; ++c) W[(size_t)c * h->cout + o] = w[(size_t)o * f + c];
            e = h->arena.upload(W, &h->fw);
            if (e == cudaSuccess) e = h->arena.upload(b, (size_t)h->cout, &h->fb);
            ok = e == cudaSuccess;
        }
    }
    if (!ok || cur.i != cur.n) {
        if (e != cudaSuccess) smk::set_error("smk_generator_create: upload failed: %s", cudaGetErrorString(e));
        else smk::set_error("smk_generator_create: consumed %d tensors but %d were given (state_dict order, num_batches_tracked removed)", cur.i, cur.n);
        delete h; return e != cudaSuccess ? (int)e : -1;
    }
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
    P.pad[0] = P.pad[1] = P.pad[2] = h->precision == 1 ? (sb + 2) * (sb + 2) * cb : 0;
    return P;
}

// One 3x3 convolution, dispatched on the handle's precision.
//   refl   : reflection padding (ResNet blocks).  At precision 1 `in` must then be a padded buffer.
//   store  : 0 plain / slice, 2 interior of a padded buffer (precision 1 only)
int conv3(const SmkGenerator* h, const Conv3& c, const float* in, int ld_in, int B, int S, bool refl, bool relu,
          const float* res, int res_pad, float* out, int ld_out, int store, cudaStream_t st, bool fuse_head = false) {
    if (c.wt) {
        TcConv p{};
        if (fuse_head) { p.head_w = h->fw; p.head_b = h->fb; p.head_c = h->cout; }
        p.in = in; p.ld_in = ld_in; p.B = B; p.H = S; p.W = S; p.Cin = c.cin_p; p.wt = c.wt; p.scale = c.scale; p.bias = c.bias;
        p.N = c.cout; p.K = 9 * c.cin_p; p.mode = refl ? 2 : 1; p.relu = relu ? 1 : 0;
        p.res = res; p.ld_res = c.cout; p.res_pad = res_pad; p.out = out; p.ld_out = ld_out; p.store = store; p.round_out = 1;
        return smk::tc_conv(p, st);
    }
    ConvProblem p{};
    p.in = in; p.ld_in = ld_in; p.B = B; p.H = S; p.W = S; p.Cin = c.cin_p;
    p.w = c.w; p.scale = c.scale; p.bias = c.bias; p.N = c.cout; p.K = 9 * c.cin_p; p.mode = refl ? 2 : 1; p.relu = relu ? 1 : 0;
    p.res = res; p.ld_res = c.cout; p.out = out; p.ld_out = ld_out; p.shuffle = 0; p.round_out = h->precision == 1 ? 1 : 0;
    return smk::conv_gemm(p, st);
}
}  // namespace

extern "C" size_t smk_generator_workspace_bytes(const SmkGenerator* h, int B) {
    return (make_plan(h).total() * (size_t)B * sizeof(float)) + 40 * 256;
}

extern "C" int smk_generator_forward(const SmkGenerator* h, const float* x, int B, float* y,
                                     void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;                      // empty batch: nothing to do (pointers may be null)
    SMK_REQUIRE(h && x && y, "smk_generator_forward: null argument");
    SMK_REQUIRE(B > 0, "smk_generator_forward: negative batch");
    SMK_REQUIRE(ws && ws_bytes >= smk_generator_workspace_bytes(h, B), "smk_generator_forward: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    smk::Workspace w(ws, ws_bytes);
    const Plan P = make_plan(h);
    const int f = h->f;
    const bool tc = h->precision == 1;
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
    int rc = smk::nchw_to_nhwc_pad(x, B, h->cin, 224, 224, h->cin_p, x8, st, tc);
    if (rc) return rc;
    // encoder levels: conv1 -> t[l]; conv2 -> upper half of cat[l] (the skip); pool -> p[l]
    const float* in = x8; int ld = h->cin_p;
    for (int l = 0; l < 4; ++l) {
        int S = 224 >> l, c = f << l;
        if ((rc = conv3(h, h->enc[l][0], in, ld, B, S, false, true, nullptr, 0, t[l], c, 0, st))) return rc;
        if ((rc = conv3(h, h->enc[l][1], t[l], c, B, S, false, true, nullptr, 0, cat[l] + c, 2 * c, 0, st))) return rc;
        if ((rc = smk::maxpool2x2(cat[l] + c, 2 * c, B, S, S, c, p[l], st))) return rc;
        in = p[l]; ld = c;
    }
    const int Sb = 14, cb = 16 * f;
    if ((rc = conv3(h, h->enc[4][0], p[3], 8 * f, B, Sb, false, true, nullptr, 0, tb, cb, 0, st))) return rc;
    const float* bott;                              // plain [B,14,14,cb] tensor feeding the first upconv
    if (!tc || h->nres == 0) {
        if ((rc = conv3(h, h->enc[4][1], tb, cb, B, Sb, false, true, nullptr, 0, b0, cb, 0, st))) return rc;
        float *cur = b0, *nxt = b1;
        for (int r = 0; r < h->nres && !tc; ++r) {  // x + BN(conv(reflpad(ReLU(BN(conv(reflpad(x)))))))
            if ((rc = conv3(h, h->res[2 * r], cur, cb, B, Sb, true, true, nullptr, 0, tb, cb, 0, st))) return rc;
            if ((rc = conv3(h, h->res[2 * r + 1], tb, cb, B, Sb, true, false, cur, 0, nxt, cb, 0, st))) return rc;
            std::swap(cur, nxt);
        }
        bott = cur;
    } else {
        // tensor-core path: residual stream lives in reflection-padded buffers  xa -> (xt) -> xb
        float *xa = pad[0], *xt = pad[1], *xb = pad[2];
        if ((rc = conv3(h, h->enc[4][1], tb, cb, B, Sb, false, true, nullptr, 0, xa, cb, 2, st))) return rc;
        if ((rc = smk::reflect_halo(xa, B, Sb, Sb, cb, st))) return rc;
        for (int r = 0; r < h->nres; ++r) {
            const bool last = r == h->nres - 1;
            if ((rc = conv3(h, h->res[2 * r], xa, cb, B, Sb, true, true, nullptr, 0, xt, cb, 2, st))) return rc;
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
        if (u.wt) {
            TcConv q{};
            q.in = din; q.ld_in = u.cin; q.B = B; q.H = dS; q.W = dS; q.Cin = u.cin; q.wt = u.wt; q.scale = u.scale; q.bias = u.bias;
            q.N = 4 * u.cout; q.K = u.cin; q.mode = 0; q.relu = 0; q.res = nullptr; q.out = cat[lvl]; q.ld_out = 2 * u.cout; q.store = 1; q.round_out = 1;
            if ((rc = smk::tc_conv(q, st))) return rc;
        } else {
            ConvProblem q{};
            q.in = din; q.ld_in = u.cin; q.B = B; q.H = dS; q.W = dS; q.Cin = u.cin; q.w = u.w; q.scale = u.scale; q.bias = u.bias;
            q.N = 4 * u.cout; q.K = u.cin; q.mode = 0; q.relu = 0; q.res = nullptr; q.ld_res = 0;
            q.out = cat[lvl]; q.ld_out = 2 * u.cout; q.shuffle = 1;
            if ((rc = smk::conv_gemm(q, st))) return rc;
        }
        dS *= 2;
        if ((rc = conv3(h, h->dec[l][0], cat[lvl], 2 * u.cout, B, dS, false, true, nullptr, 0, t[lvl], u.cout, 0, st))) return rc;
        // last layer of the tensor-core path: the 1x1 conv + sigmoid (smirk_generator.py:77-78,86) rides in the epilogue of
        // dec1conv2 — the [B,224,224,32] activation (6.4 MB per face) is neither written nor read back
        const bool fuse_head = l == 3 && tc && u.cout <= 32;
        if (fuse_head) return conv3(h, h->dec[l][1], t[lvl], u.cout, B, dS, false, true, nullptr, 0, y, u.cout, 3, st, true);
        if ((rc = conv3(h, h->dec[l][1], t[lvl], u.cout, B, dS, false, true, nullptr, 0, d[lvl], u.cout, 0, st))) return rc;
        din = d[lvl];
    }
    return smk::conv1x1_sigmoid_nchw(d[0], B, 224 * 224, f, h->fw, h->fb, h->cout, y, st);
}
