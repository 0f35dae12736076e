// SmirkEncoder forward: three MobileNetV3-"minimal" backbones + pooled linear heads.
//
// Replaces SmirkEncoder.forward (reference src/smirk_encoder.py:123-133) including the timm backbones
// built at :7-12 (tf_mobilenetv3_small_minimal_100 for pose, ..._large_minimal_100 for shape and
// expression; ReLU only, no squeeze-excite, 3x3 depthwise, BN eps 1e-3, TF-SAME padding) and the
// heads/clamps at :34-45, :66-73, :95-110.  BatchNorm (eval mode) is folded into a per-channel
// scale/bias applied in each convolution's epilogue; activations live in NHWC fp32.
//
// Input gradient (frozen weights, eval BN): smk_encoder_forward_saved runs the forward's launches and also keeps the
// output of every ReLU and the pre-clamp head values in a caller-owned `saved` buffer (layers that write to HBM anyway
// write there directly; the fused stem + block 0 and expand + depthwise kernels and the pooled head store a second copy
// behind a template flag).  smk_encoder_backward walks each backbone backwards: head (clamp masks, pooled linear, the
// `cn` ReLU), 1x1 dgrads as ordinary GEMMs over weights (diag(s) W)^T packed at create time (the folded BN scale rides in
// the weights), a CUDA-core depthwise dgrad that applies both ReLU masks of its block, and one transposed stem conv that
// sums the backbones' gradients into the NCHW image gradient.
#include "encoder.cuh"
#include "nn_kernels.cuh"
#include "gemm_tc.cuh"
#include "xdw_tc.cuh"
#include "../../include/smirk_b200_live.h"
#include <math.h>

namespace {

using namespace enc;
using smk::TensorCursor;
using smk::grid_of;
using smk::same_pad_begin;

constexpr float kBnEps = 1e-3f;

// The operands of one conv, decided once for the host fold (smk_encoder_create) and the device refresh
// (smk_encoder_live_create):
//   kind 0 = 1x1 [Cout,Cin,1,1]: smk::pack_gemm operands, the forward's N = cout, K = cin, the dgrad's (diag(s) W)^T,
//            N = cin, K = cout.  fwd_tc / dgrad_tc: TF32 [N][K] (with tails when x3), otherwise fp32 [K][N]; the forward
//            is fp32 even when tc for a DS block's 1x1 that stem_ds runs (fwd_f32).
//   kind 1 = depthwise [C,1,3,3] -> W[9][C]; dgrad: flipped taps, Wd[8 - k][c] = s[c] W[c][k]
//   kind 2 = stem [16,3,3,3] -> W[27][16]; dgrad: Wd[k][o] = s[o] W[o][k] (the forward layout)
struct ConvOps { int kind, cin, cout; bool fwd_tc, dgrad_tc, x3; };
ConvOps conv_ops(int kind, int cin, int cout, bool tc, bool x3, bool fwd_f32 = false) {
    const bool pw = kind == 0;
    return ConvOps{kind, cin, cout, pw && tc && !fwd_f32, pw && tc, pw && tc && x3};
}

// Consumes (conv weight, bn gamma, beta, mean, var) from the tensor list: the folded BN scale s and bias, the forward
// weights, and the dgrad weights, which carry s.
bool fold_conv(TensorCursor& cur, const ConvOps& c, smk::DeviceArena& arena, ConvW* out, cudaError_t* err) {
    const float* w = cur.next(); const float* g = cur.next(); const float* b = cur.next();
    const float* mu = cur.next(); const float* var = cur.next();
    if (!w || !g || !b || !mu || !var) return false;
    const int cin = c.cin, cout = c.cout, kind = c.kind;
    std::vector<float> S(cout), Bi(cout);
    smk::fold_bn(g, b, mu, var, cout, kBnEps, S.data(), Bi.data());
    out->cin = cin; out->cout = cout;
    cudaError_t e = arena.upload(S, &out->scale);
    if (e == cudaSuccess) e = arena.upload(Bi, &out->bias);
    if (kind == 0) {                                          // torch's [Cout][Cin] is the forward's [N][K]
        if (e == cudaSuccess) e = smk::pack_gemm(arena, cout, cin, c.fwd_tc, c.x3, w, &out->fwd);
        if (e == cudaSuccess) e = smk::pack_gemm(arena, cin, cout, c.dgrad_tc, c.x3, [&](int ci, int o) { return S[o] * w[(size_t)o * cin + ci]; }, &out->dgrad);
    } else {
        const int K = kind == 1 ? 9 : 27;
        std::vector<float> W((size_t)K * cout), D(W.size());
        for (int o = 0; o < cout; ++o)
            for (int k = 0; k < K; ++k) {
                W[(size_t)k * cout + o] = w[(size_t)o * K + k];
                D[(size_t)(kind == 1 ? 8 - k : k) * cout + o] = S[o] * w[(size_t)o * K + k];
            }
        float *fw = nullptr, *dw = nullptr;
        if (e == cudaSuccess) e = arena.upload(W, &fw);
        if (e == cudaSuccess) e = arena.upload(D, &dw);
        out->fwd = smk::GemmW{fw, nullptr, nullptr}; out->dgrad = smk::GemmW{dw, nullptr, nullptr};
    }
    *err = e;
    return e == cudaSuccess;
}

// The live counterpart of fold_conv for the conv whose weight is tensor t of backbone i: allocates its buffers and records
// the refresh's fold and pack jobs in the layouts of fold_conv (trn::PackJob: MAT transposes torch's [cout][cols] where
// the operand is not torch-ordered, DW_DGRAD flips the depthwise taps; the dgrad jobs multiply in the folded scale).
cudaError_t live_conv(const ConvOps& c, int i, int t, smk::DeviceArena& arena, trn::LivePlan& plan, ConvW* out) {
    const int cin = c.cin, cout = c.cout, cols = c.kind == 0 ? cin : c.kind == 1 ? 9 : 27;
    out->cin = cin; out->cout = cout;
    cudaError_t e = arena.alloc((size_t)cout, &out->scale);
    if (e == cudaSuccess) e = arena.alloc((size_t)cout, &out->bias);
    if (e != cudaSuccess) return e;
    plan.folds.push_back(trn::LiveFold{i, t, trn::FoldJob{nullptr, nullptr, nullptr, nullptr, out->scale, out->bias, cout, 0.f}});
    // One operand of torch's [cout][cols] weight: transposed unless torch-ordered, split into TF32 heads (+ tails) when tc.
    auto add = [&](int kind, bool transpose, bool tc, const float* scale, smk::GemmW* w) {
        trn::PackJob j{};
        j.kind = kind; j.rows = cout; j.cols = cols; j.transpose = transpose ? 1 : 0; j.split = tc ? 1 : 0; j.cout = cout; j.scale = scale;
        const size_t n = (size_t)cout * cols;
        float *hi = nullptr, *lo = nullptr;
        cudaError_t r = arena.alloc(n, &hi);
        if (r == cudaSuccess && tc && c.x3) r = arena.alloc(n, &lo);
        j.hi = hi; j.lo = lo;
        plan.jobs.push_back(trn::LiveJob{i, t, j});
        plan.bytes += 4.0 * n * (2 + (lo ? 1 : 0));
        *w = tc ? smk::GemmW{nullptr, hi, lo} : smk::GemmW{hi, nullptr, nullptr};
        return r;
    };
    if (c.kind == 0) {          // forward [N = cout][K = cin] is torch's order; the dgrad's [N = cin][K = cout] is its transpose
        e = add(trn::MAT, !c.fwd_tc, c.fwd_tc, nullptr, &out->fwd);
        if (e == cudaSuccess) e = add(trn::MAT, c.dgrad_tc, c.dgrad_tc, out->scale, &out->dgrad);
    } else {                    // fp32 [K][N] = torch's [cout][K] transposed; the depthwise dgrad flips its taps
        e = add(trn::MAT, true, false, nullptr, &out->fwd);
        if (e == cudaSuccess) e = add(c.kind == 1 ? trn::DW_DGRAD : trn::MAT, c.kind != 1, false, out->scale, &out->dgrad);
    }
    return e;
}

// Stem + block 0 run as one fp32 kernel (stem_ds) at every precision but 1, whose block-0 1x1 runs on TF32 tensor cores.
bool fuse_stem(const SmkEncoder* h) { return h->precision == 0 || h->fuse_xdw; }

// Every conv of backbone i in tensor-list order with its operands: visit(ConvOps, ConvW*) -> false stops the walk.
template <typename Visit>
bool for_each_conv(SmkEncoder* h, int i, Visit&& visit) {
    const bool tc = h->precision >= 1, x3 = h->x3;
    Backbone& bb = h->bb[i];
    if (!visit(conv_ops(2, 3, 16, false, false), &bb.stem)) return false;
    for (Block& b : bb.blocks) {
        bool ok;
        if (b.kind == DS) ok = visit(conv_ops(1, b.cin, b.cin, false, false), &b.dw) && visit(conv_ops(0, b.cin, b.cout, tc, x3, fuse_stem(h)), &b.pw);
        else if (b.kind == IR) ok = visit(conv_ops(0, b.cin, b.mid, tc, x3), &b.pw) && visit(conv_ops(1, b.mid, b.mid, false, false), &b.dw) &&
                                    visit(conv_ops(0, b.mid, b.cout, tc, x3), &b.pwl);
        else ok = visit(conv_ops(0, b.cin, b.cout, tc, x3), &b.pw);
        if (!ok) return false;
    }
    return true;
}

// The saved-tensor layout of backbone i's eval path: forward order (names: the reference's module paths).
void add_saved(SmkEncoder* h, int i) {
    Backbone& bb = h->bb[i];
    auto add = [h](const std::string& name, int H, int C) { return h->saved.add(name, H, H, C); };
    bb.sv_stem = add(std::string(kEncName[i]) + ".encoder.bn1", 112, 16);
    for (Block& b : bb.blocks) {
        if (b.kind == DS) b.sv_a = add(b.path + ".bn1", b.hout, b.cin);
        else if (b.kind == IR) { b.sv_a = add(b.path + ".bn1", b.hin, b.mid); b.sv_b = add(b.path + ".bn2", b.hout, b.mid); }
        else b.sv_a = add(b.path + ".bn1", b.hout, b.cout);
    }
    bb.sv_head = add(std::string(kEncName[i]) + "." + kHeadName[i], 1, bb.n_out);
}

// Precision 0-3 of SmkEncoderDesc -> the handle's flags.
void set_precision(SmkEncoder* h, int precision) {
    h->precision = precision >= 1 ? 1 : 0; h->fuse_xdw = precision >= 2; h->x3 = precision == 3;
}

// A handle refreshed on the device must have been refreshed once before the eval path reads its weights.
#define SMK_REQUIRE_WEIGHTS(h, fn) \
    SMK_REQUIRE(!(h)->live || (h)->refreshed, "%s: a live handle whose weights were never set: call smk_encoder_refresh first", fn)

}  // namespace

extern "C" int smk_encoder_create(const SmkEncoderDesc* desc, SmkEncoder** out) {
    SMK_REQUIRE(desc && out, "smk_encoder_create: null argument");
    SMK_REQUIRE(desc->precision >= 0 && desc->precision <= 3,
                "smk_encoder_create: precision must be 0 (fp32 CUDA cores), 1 (tf32 wgmma 1x1 convs), 2 (1 + fused expand/depthwise blocks) or "
                "3 (2 with 3xTF32 error-compensated tensor-core arithmetic: fp32-equivalent results)");
    if (desc->precision >= 1) { if (int rc = smk::tc_init()) return rc; }
    SmkEncoder* h = new SmkEncoder();
    h->n_shape = desc->n_shape; h->n_exp = desc->n_exp;
    set_precision(h, desc->precision);
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 3; ++i) {
        Backbone& bb = h->bb[i];
        if (desc->n_tensors[i] == 0 || desc->tensors[i] == nullptr) continue;        // backbone not part of this handle
        h->present[i] = true;
        build_backbone(h, i);
        TensorCursor cur{desc->tensors[i], desc->n_tensors[i]};
        const bool ok = for_each_conv(h, i, [&](const ConvOps& c, ConvW* w) { return fold_conv(cur, c, h->arena, w, &e); });
        if (!ok || cur.i != cur.n) {
            if (e != cudaSuccess) smk::set_error("smk_encoder_create: upload failed: %s", cudaGetErrorString(e));
            else smk::set_error("smk_encoder_create: backbone %d expects %d tensors (conv weight + 4 BN tensors per conv), got %d",
                                i, cur.i, cur.n);
            delete h; return e != cudaSuccess ? (int)e : -1;
        }
        e = h->arena.upload(desc->head_w[i], (size_t)bb.n_out * bb.feat, &bb.head_w);
        if (e == cudaSuccess) e = h->arena.upload(desc->head_b[i], (size_t)bb.n_out, &bb.head_b);
        if (e != cudaSuccess) { smk::set_error("smk_encoder_create: upload failed: %s", cudaGetErrorString(e)); delete h; return (int)e; }
        add_saved(h, i);
    }
    if (!h->present[0] && !h->present[1] && !h->present[2]) { smk::set_error("smk_encoder_create: no backbone given"); delete h; return -1; }
    e = finish_create(h);
    if (e != cudaSuccess) { smk::set_error("smk_encoder_create: upload or stream/event creation failed: %s", cudaGetErrorString(e)); delete h; return (int)e; }
    *out = h;
    return 0;
}

extern "C" int smk_encoder_live_create(int backbones, int n_shape, int n_exp, int precision, SmkEncoder** out) {
    SMK_REQUIRE(out, "smk_encoder_live_create: null argument");
    SMK_REQUIRE(backbones > 0 && backbones < 8, "smk_encoder_live_create: backbones is a non-empty bit set of {1 pose, 2 shape, 4 expression}");
    SMK_REQUIRE(precision >= 0 && precision <= 3, "smk_encoder_live_create: precision must be 0, 1, 2 or 3");
    SMK_REQUIRE(n_shape > 0 && n_exp >= 0 && n_shape <= 4096 && n_exp <= 4096, "smk_encoder_live_create: bad head widths");
    if (precision >= 1) { if (int rc = smk::tc_init()) return rc; }
    SmkEncoder* h = new SmkEncoder();
    h->live = true;
    h->n_shape = n_shape; h->n_exp = n_exp;
    set_precision(h, precision);
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 3 && e == cudaSuccess; ++i) {
        if (!((backbones >> i) & 1)) continue;
        Backbone& bb = h->bb[i];
        h->present[i] = true;
        build_backbone(h, i);
        int t = 0;
        for_each_conv(h, i, [&](const ConvOps& c, ConvW* w) { e = live_conv(c, i, t, h->arena, h->plan, w); t += 5; return e == cudaSuccess; });
        h->live_tensors[i] = t;
        for (int k = 0; k < 2 && e == cudaSuccess; ++k) {             // the heads, copied as they are
            float* dst = nullptr;
            const int n = k == 0 ? bb.n_out * bb.feat : bb.n_out;
            e = h->arena.alloc((size_t)n, &dst);
            trn::PackJob j{};
            j.kind = trn::MAT; j.rows = 1; j.cols = n; j.hi = dst;
            h->plan.jobs.push_back(trn::LiveJob{i, -1 - k, j});
            h->plan.bytes += 8.0 * n;
            (k == 0 ? bb.head_w : bb.head_b) = dst;
        }
        add_saved(h, i);
    }
    if (e == cudaSuccess) e = finish_create(h);
    if (e != cudaSuccess) { smk::set_error("smk_encoder_live_create: allocation or stream/event creation failed: %s", cudaGetErrorString(e)); delete h; return (int)e; }
    *out = h;
    return 0;
}

extern "C" int smk_encoder_refresh(SmkEncoder* h, const SmkEncoderTrainArgs* a, void* stream) {
    const char* fn = "smk_encoder_refresh";
    SMK_REQUIRE(h && h->live, "%s: not a live handle (smk_encoder_live_create)", fn);
    SMK_REQUIRE(a, "%s: null args", fn);
    for (int i = 0; i < 3; ++i) {
        if (!h->present[i]) continue;
        const int n = h->live_tensors[i];
        SMK_REQUIRE(a->tensors[i] && a->n_tensors[i] == n, "%s: backbone %d expects %d tensors (conv weight + 4 BN tensors per conv), got %d",
                    fn, i, n, a->n_tensors[i]);
        for (int k = 0; k < n; ++k) SMK_REQUIRE(a->tensors[i][k], "%s: backbone %d: null tensor %d", fn, i, k);
        SMK_REQUIRE(a->head_w[i] && a->head_b[i], "%s: backbone %d: null head", fn, i);
        SMK_REQUIRE(a->eps[i] > 0.f, "%s: backbone %d: eps must be positive", fn, i);
    }
    const float* const* t[3] = {a->tensors[0], a->tensors[1], a->tensors[2]};
    if (int rc = trn::refresh(h->plan, t, a->head_w, a->head_b, a->eps, (cudaStream_t)stream)) return rc;
    h->refreshed = true;
    return 0;
}

extern "C" void smk_encoder_destroy(SmkEncoder* h) { delete h; }

extern "C" size_t smk_encoder_workspace_bytes(const SmkEncoder* h, int B) {
    return 12 * smk::ws_round((size_t)B * h->max_act * sizeof(float));      // 4 buffers per backbone, 3 concurrent backbones
}

// One 1x1 convolution for n = 1 or 2 backbones of identical structure (c[k], in[k], res[k], out[k]).  On the tensor-core
// path a pair shares ONE launch (gemm_tc.cu, TcMaps): half the launches and twice the tiles per launch for layers that
// sit on the launch/latency floor.  Backbones are paired only on the tensor-core path.
static int pointwise(int n, const ConvW* const* c, float* const* in, int B, int H, int W, bool relu, float* const* res, float* const* out, cudaStream_t st) {
    smk::Conv q[2];
    for (int k = 0; k < n; ++k) {
        q[k] = smk::Conv{};
        q[k].in = in[k]; q[k].ld_in = c[k]->cin; q[k].B = B; q[k].H = H; q[k].W = W; q[k].Cin = c[k]->cin;
        q[k].wgt = c[k]->fwd; q[k].scale = c[k]->scale; q[k].bias = c[k]->bias;
        q[k].N = c[k]->cout; q[k].K = c[k]->cin; q[k].mode = 0; q[k].relu = relu ? 1 : 0;
        q[k].res = res ? res[k] : nullptr; q[k].ld_res = c[k]->cout; q[k].out = out[k]; q[k].ld_out = c[k]->cout;
        q[k].round_out = c[k]->fwd.wt && !c[k]->fwd.wt_lo;      // 3xTF32 consumers split full fp32 activations themselves
    }
    return smk::conv(q[0], st, n == 2 ? &q[1] : nullptr);
}

// The forward; sv (grad mode, may be null): the saved buffer.  With sv the launches and arithmetic are those of the
// forward-only path: the ReLU outputs the forward writes to HBM anyway (stem, unfused e / d, cn) go to their saved slot
// instead of a workspace buffer, the fused kernels and the head store a second copy.
static int encoder_forward(const SmkEncoder* h, const float* img, int B, float* pose_cam, float* shape, float* expr, float* sv,
                           void* ws, size_t ws_bytes, cudaStream_t main_st) {
    smk::Workspace w(ws, ws_bytes);
    float* bufs[3][4];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 4; ++j) bufs[i][j] = w.take<float>((size_t)B * h->max_act);
    SMK_REQUIRE(bufs[2][3] != nullptr, "smk_encoder_forward: workspace carve-up failed");
    float* outs[3] = {pose_cam, shape, expr};
    auto SV = [&](int i) -> float* { return sv ? sv + (size_t)B * h->saved.off[i] : nullptr; };
    const bool fused = fuse_stem(h);
    const bool rnd = h->precision == 1 && !h->x3;                 // activations that feed a plain TF32 layer are rounded
    // Before the fork, on main_st, one pass over the image (the only tensor the backbones share) for every backbone: stem
    // + block 0 (depthwise-separable, 16 channels at 112 x 112) as one kernel, so the three largest activations never
    // reach HBM and each unit's walk starts at block 1; at precision 1 the stems alone.
    float* in0[3];                        // what the walk's first block reads: block 0's output, or the stem's
    smk::StemDsProblem sp[3];
    smk::StemProblem sq[3];
    int n_present = 0;
    for (int i = 0; i < 3; ++i) {
        if (!h->present[i]) continue;
        const Backbone& bb = h->bb[i];
        const Block& b0 = bb.blocks[0];
        in0[i] = sv && !fused ? SV(bb.sv_stem) : bufs[i][0];
        sp[n_present] = smk::StemDsProblem{bb.stem.fwd.w, bb.stem.scale, bb.stem.bias, b0.dw.fwd.w, b0.dw.scale, b0.dw.bias,
                                           b0.pw.fwd.w, b0.pw.scale, b0.pw.bias, in0[i], SV(bb.sv_stem), SV(b0.sv_a), b0.stride};
        sq[n_present++] = smk::StemProblem{bb.stem.fwd.w, bb.stem.scale, bb.stem.bias, in0[i]};
    }
    if (int rc = fused ? smk::stem_ds(img, B, 224, 224, sp, n_present, rnd ? 1 : 0, main_st)
                       : smk::stem_conv(img, B, 224, 224, sq, n_present, main_st)) return rc;
    return for_each_unit(h, h->present, main_st, "smk_encoder_forward", [&](const Unit& unit) {
        const int n = unit.n;
        cudaStream_t st = unit.st;
        int rc = 0;
        // x / y: the workspace ping-pong pair; cur: the current block's input (x, or a saved tensor)
        const Backbone* bb[2]; float *x[2], *y[2], *e[2], *d[2], *cur[2];
        for (int k = 0; k < n; ++k) {
            const int i = unit.idx[k];
            bb[k] = &h->bb[i]; x[k] = bufs[i][0]; y[k] = bufs[i][1]; e[k] = bufs[i][2]; d[k] = bufs[i][3]; cur[k] = in0[i];
        }
        const size_t first = fused ? 1 : 0;
        int res = 112 / (fused ? bb[0]->blocks[0].stride : 1);
        for (size_t bi = first; bi < bb[0]->blocks.size() && !rc; ++bi) {
            const Block* b[2] = {&bb[0]->blocks[bi], &bb[n - 1]->blocks[bi]};
            const Block& b0 = *b[0];
            const int ro = (res + b0.stride - 1) / b0.stride;
            const ConvW* pw[2] = {&b[0]->pw, &b[1]->pw};
            const ConvW* pwl[2] = {&b[0]->pwl, &b[1]->pwl};
            float* out[2] = {y[0], y[1]};                // the block's output
            if (sv) {                                    // saved ReLU outputs the forward writes to HBM anyway
                for (int k = 0; k < n; ++k) {
                    if (b0.kind == DS) d[k] = SV(b[k]->sv_a);
                    else if (b0.kind == IR) { e[k] = SV(b[k]->sv_a); d[k] = SV(b[k]->sv_b); }
                    else out[k] = SV(b[k]->sv_a);
                }
            }
            if (b0.kind == DS) {                         // block 0 at precision 1 (stem_ds runs it at the others)
                for (int k = 0; k < n && !rc; ++k)
                    rc = smk::dwconv3x3(cur[k], B, res, res, b[k]->cin, b[k]->stride, b[k]->dw.fwd.w, b[k]->dw.scale, b[k]->dw.bias, d[k], st, rnd);
                if (!rc) rc = pointwise(n, pw, d, B, ro, ro, false, b0.skip ? cur : nullptr, out, st);
            } else if (b0.kind == IR) {
                // The 7x7 layers (a 16x16 window holds 81 useful pixels, 49 outputs) run as 1x1 GEMM + depthwise kernels:
                // most of a window would be halo; every other resolution runs fused.
                constexpr int kXdwMinRes = 8;
                if (h->fuse_xdw && b0.pw.fwd.wt && res >= kXdwMinRes) {
                    // expand 1x1 + depthwise 3x3 in one kernel: the expanded tensor never leaves the SM
                    smk::XdwConv q[2];
                    for (int k = 0; k < n; ++k) {
                        q[k] = smk::XdwConv{};
                        q[k].x = cur[k]; q[k].B = B; q[k].H = res; q[k].W = res; q[k].Cin = b[k]->cin; q[k].w1t = b[k]->pw.fwd.wt; q[k].w1t_lo = b[k]->pw.fwd.wt_lo;
                        q[k].scale1 = b[k]->pw.scale; q[k].bias1 = b[k]->pw.bias; q[k].mid = b[k]->mid; q[k].wdw = b[k]->dw.fwd.w;
                        q[k].scale2 = b[k]->dw.scale; q[k].bias2 = b[k]->dw.bias; q[k].stride = b[k]->stride; q[k].round_out = h->x3 ? 0 : 1; q[k].out = d[k];
                        q[k].e_out = sv ? e[k] : nullptr;
                    }
                    rc = smk::xdw_conv(q[0], st, n == 2 ? &q[1] : nullptr);
                } else {
                    rc = pointwise(n, pw, cur, B, res, res, true, nullptr, e, st);
                    for (int k = 0; k < n && !rc; ++k)
                        rc = smk::dwconv3x3(e[k], B, res, res, b[k]->mid, b[k]->stride, b[k]->dw.fwd.w, b[k]->dw.scale, b[k]->dw.bias, d[k], st, rnd);
                }
                if (!rc) rc = pointwise(n, pwl, d, B, ro, ro, false, b0.skip ? cur : nullptr, out, st);
            } else {
                rc = pointwise(n, pw, cur, B, res, res, true, nullptr, out, st);
            }
            if (rc) break;
            for (int k = 0; k < n; ++k) {
                cur[k] = out[k];
                if (out[k] == y[k]) std::swap(x[k], y[k]);      // x now holds the block output, y is free
            }
            res = ro;
        }
        if (!rc) {                              // global average pool + head + clamps: one launch per unit
            smk::GapHeadProblem gp[2];
            for (int k = 0; k < n; ++k)
                gp[k] = smk::GapHeadProblem{cur[k], bb[k]->head_w, bb[k]->head_b, bb[k]->codes, outs[unit.idx[k]], bb[k]->n_out,
                                            SV(bb[k]->sv_head)};
            rc = smk::gap_head(gp, n, B, res * res, bb[0]->feat, st);
        }
        return rc;
    });
}

extern "C" int smk_encoder_forward(const SmkEncoder* h, const float* img, int B, float* pose_cam, float* shape,
                                   float* expr, void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;                      // empty batch: nothing to do (pointers may be null)
    SMK_REQUIRE(h && img, "smk_encoder_forward: null argument");
    SMK_REQUIRE((pose_cam || !h->present[0]) && (shape || !h->present[1]) && (expr || !h->present[2]),
                "smk_encoder_forward: null output for a backbone this handle holds");
    SMK_REQUIRE(B > 0, "smk_encoder_forward: negative batch");
    SMK_REQUIRE(ws && ws_bytes >= smk_encoder_workspace_bytes(h, B), "smk_encoder_forward: workspace too small");
    SMK_REQUIRE(!h->train, "smk_encoder_forward: a train-mode handle runs smk_encoder_forward_train");
    SMK_REQUIRE_WEIGHTS(h, "smk_encoder_forward");
    return encoder_forward(h, img, B, pose_cam, shape, expr, nullptr, ws, ws_bytes, (cudaStream_t)stream);
}

// ---- input gradient --------------------------------------------------------------------------------------------------
namespace {

// Head backward for one or two backbones (blockIdx.z): g_p = g_out * [clamp / ReLU passes p] (torch: clamp passes on
// [lo, hi] inclusive, relu where p > 0), g_feat = W^T g_p / HW, broadcast over the HW pixels of the map and masked by the
// saved `cn` output -> the gradient of the cn pre-activation, [B, HW, C].  CTA = (image, 256 channels).
struct HeadBwd { const float* g[2]; const float* raw[2]; const uint8_t* codes[2]; const float* w[2]; const float* cn[2]; float* out[2]; int n_out[2]; };
__global__ void __launch_bounds__(256)
head_bwd_kernel(const __grid_constant__ HeadBwd p, int HW, int C, int round) {
    extern __shared__ float gp[];                     // [n_out]
    const int q = blockIdx.z, b = blockIdx.x, n_out = p.n_out[q];
    const uint8_t* codes = p.codes[q];
    for (int o = threadIdx.x; o < n_out; o += blockDim.x) {
        const float v = p.raw[q][(size_t)b * n_out + o];
        const int code = codes ? codes[o] : 0;
        const bool pass = code == 1 ? (v >= 0.f && v <= 1.f) : code == 2 ? v > 0.f : code == 3 ? (v >= -0.2f && v <= 0.2f) : true;
        gp[o] = pass ? p.g[q][(size_t)b * n_out + o] : 0.f;
    }
    __syncthreads();
    const int c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const float* w = p.w[q];
    float acc = 0.f;
    for (int o = 0; o < n_out; ++o) acc = fmaf(__ldg(w + (size_t)o * C + c), gp[o], acc);
    const float gf = acc * (1.f / (float)HW);
    const float* m = p.cn[q] + (size_t)b * HW * C + c;
    float* out = p.out[q] + (size_t)b * HW * C + c;
    for (int px = 0; px < HW; ++px) {
        float v = __ldg(m + (size_t)px * C) > 0.f ? gf : 0.f;
        out[(size_t)px * C] = round ? smk::round_tf32(v) : v;
    }
}

// Depthwise dgrad for one or two backbones (blockIdx.z): the exact adjoint of dwconv3x3 (TF-SAME, pad_begin `pad`; stride 2
// pads bottom / right only on the even maps used here), with both ReLU masks of the block:
//   out[ih, iw, c] = [a[ih, iw, c] > 0] * (sum_taps wf[tap][c] * [d > 0] * g (oh, ow) + res[ih, iw, c])
// wf: flipped taps with the folded BN scale (fold_conv), g / d: [B, Ho, Wo, C] gradient of the depthwise output and the
// saved output, a: the saved block input (IR: e, DS: the stem output), res: optional (the DS skip).  Thread = (pixel, quad).
struct DwDgrad { const float* g[2]; const float* d[2]; const float* a[2]; const float* res[2]; const float* w[2]; float* out[2]; };
template <int STRIDE>
__global__ void __launch_bounds__(256)
dw_dgrad_kernel(const __grid_constant__ DwDgrad p, int B, int H, int W, int C, int Ho, int Wo, int pad, int round) {
    const int q = blockIdx.z, C4 = C >> 2;
    const float4* g = reinterpret_cast<const float4*>(p.g[q]);
    const float4* d = reinterpret_cast<const float4*>(p.d[q]);
    const float4* wf = reinterpret_cast<const float4*>(p.w[q]);
    const long total = (long)B * H * W * C4;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4); const long pix = i / C4;
        const int iw = (int)(pix % W); const long t = pix / W; const int ih = (int)(t % H); const int b = (int)(t / H);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 3; ++j) {                 // flipped row tap j = 2 - ky
            const int ny = ih + pad - 2 + j;
            if (ny < 0 || ny % STRIDE) continue;
            const int oh = ny / STRIDE;
            if (oh >= Ho) continue;
#pragma unroll
            for (int jx = 0; jx < 3; ++jx) {
                const int nx = iw + pad - 2 + jx;
                if (nx < 0 || nx % STRIDE) continue;
                const int ow = nx / STRIDE;
                if (ow >= Wo) continue;
                const size_t o = (((size_t)b * Ho + oh) * Wo + ow) * C4 + c4;
                const float4 gv = __ldg(g + o), dv = __ldg(d + o), k = __ldg(wf + (size_t)(j * 3 + jx) * C4 + c4);
                acc.x = fmaf(dv.x > 0.f ? gv.x : 0.f, k.x, acc.x); acc.y = fmaf(dv.y > 0.f ? gv.y : 0.f, k.y, acc.y);
                acc.z = fmaf(dv.z > 0.f ? gv.z : 0.f, k.z, acc.z); acc.w = fmaf(dv.w > 0.f ? gv.w : 0.f, k.w, acc.w);
            }
        }
        if (p.res[q]) {
            const float4 r = __ldg(reinterpret_cast<const float4*>(p.res[q]) + i);
            acc.x += r.x; acc.y += r.y; acc.z += r.z; acc.w += r.w;
        }
        const float4 a = __ldg(reinterpret_cast<const float4*>(p.a[q]) + i);
        acc.x = a.x > 0.f ? acc.x : 0.f; acc.y = a.y > 0.f ? acc.y : 0.f; acc.z = a.z > 0.f ? acc.z : 0.f; acc.w = a.w > 0.f ? acc.w : 0.f;
        if (round) { acc.x = smk::round_tf32(acc.x); acc.y = smk::round_tf32(acc.y); acc.z = smk::round_tf32(acc.z); acc.w = smk::round_tf32(acc.w); }
        reinterpret_cast<float4*>(p.out[q])[i] = acc;
    }
}

// Stem dgrad: the transposed 3x3 stride-2 conv (TF-SAME) of each backbone's stem pre-activation gradient g [B, Hs, Ws, 16]
// with its scaled weights w [27][16], summed over the backbones in slot order (pose, shape, expression) straight into the
// NCHW image gradient.  A null g skips its backbone; with all three null the output is zero.  Thread = image pixel.
struct StemDgrad { const float* g[3]; const float* w[3]; };
__global__ void __launch_bounds__(128)
stem_dgrad_kernel(const __grid_constant__ StemDgrad p, int B, int H, int W, int Hs, int Ws, int pad, float* __restrict__ out) {
    __shared__ __align__(16) float sw[3][27 * 16];
    for (int k = 0; k < 3; ++k)
        if (p.w[k]) for (int i = threadIdx.x; i < 27 * 16; i += blockDim.x) sw[k][i] = p.w[k][i];
    __syncthreads();
    const long pix = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= (long)B * H * W) return;
    const int iw = (int)(pix % W); const long t = pix / W; const int ih = (int)(t % H); const int b = (int)(t / H);
    float acc[3] = {0.f, 0.f, 0.f};
    for (int k = 0; k < 3; ++k) {
        if (!p.g[k]) continue;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int ny = ih + pad - ky;
            if (ny < 0 || (ny & 1) || (ny >> 1) >= Hs) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int nx = iw + pad - kx;
                if (nx < 0 || (nx & 1) || (nx >> 1) >= Ws) continue;
                const float4* gv = reinterpret_cast<const float4*>(p.g[k] + (((size_t)b * Hs + (ny >> 1)) * Ws + (nx >> 1)) * 16);
                float gs[16];
#pragma unroll
                for (int v = 0; v < 4; ++v) { const float4 x = __ldg(gv + v); gs[4 * v] = x.x; gs[4 * v + 1] = x.y; gs[4 * v + 2] = x.z; gs[4 * v + 3] = x.w; }
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float* wk = sw[k] + ((c * 3 + ky) * 3 + kx) * 16;
#pragma unroll
                    for (int o = 0; o < 16; ++o) acc[c] = fmaf(gs[o], wk[o], acc[c]);
                }
            }
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) out[(((size_t)b * 3 + c) * H + ih) * W + iw] = acc[c];
}

// 1x1 dgrad of n = 1 or 2 backbones over their convs' dgrad weights: out[m, :N] = g[m, :K] . Wd (+ res), K = the conv's
// cout, N = its cin.
int dgrad_pw(const SmkEncoder* h, int n, const ConvW* const* c, const float* const* g, int B, int H, int W, const float* const* res,
             float* const* out, bool round, const char* tag, cudaStream_t st) {
    smk::Conv q[2];
    for (int k = 0; k < n; ++k) {
        q[k] = smk::Conv{};
        q[k].in = g[k]; q[k].ld_in = c[k]->cout; q[k].B = B; q[k].H = H; q[k].W = W; q[k].Cin = c[k]->cout;
        q[k].wgt = c[k]->dgrad; q[k].scale = h->ones; q[k].bias = h->zeros;
        q[k].N = c[k]->cin; q[k].K = c[k]->cout; q[k].mode = 0;
        q[k].res = res ? res[k] : nullptr; q[k].ld_res = c[k]->cin; q[k].out = out[k]; q[k].ld_out = c[k]->cin;
        q[k].round_out = round ? 1 : 0; q[k].tag = tag;
    }
    return smk::conv(q[0], st, n == 2 ? &q[1] : nullptr);
}

int dgrad_dw(int n, const Block* const* b, const float* const* g, const float* const* d, const float* const* a, const float* const* res,
             int B, int H, float* const* out, bool round, cudaStream_t st) {
    DwDgrad p{};
    for (int k = 0; k < 2; ++k) {
        const int j = k < n ? k : n - 1;
        p.g[k] = g[j]; p.d[k] = d[j]; p.a[k] = a[j]; p.res[k] = res ? res[j] : nullptr; p.w[k] = b[j]->dw.dgrad.w; p.out[k] = out[j];
    }
    const int C = b[0]->mid, S = b[0]->stride, Ho = (H + S - 1) / S;
    SMK_REQUIRE(C % 4 == 0 && (S == 1 || H % 2 == 0), "dw_dgrad: C must be a multiple of 4 and stride-2 maps even");
    const long total = (long)B * H * H * (C / 4);
    SMK_TAG(smk::g_prof_detail ? smk::prof_shape_tag("dw_dgrad", (long)B * H * H, S, C) : "dw_dgrad",
            n * 4.0 * ((double)B * H * H * C * (2 + (res ? 1 : 0)) + 2.0 * B * Ho * Ho * C + 9.0 * C), n * 18.0 * B * Ho * Ho * C, st);
    if (S == 1) SMK_LAUNCH(dw_dgrad_kernel<1>, dim3(grid_of(total), 1, n), dim3(256), 0, st, p, B, H, H, C, Ho, Ho, same_pad_begin(H, 1), round ? 1 : 0);
    else SMK_LAUNCH(dw_dgrad_kernel<2>, dim3(grid_of(total), 1, n), dim3(256), 0, st, p, B, H, H, C, Ho, Ho, same_pad_begin(H, 2), round ? 1 : 0);
    SMK_CHECK_LAUNCH();
    return 0;
}

}  // namespace

extern "C" size_t smk_encoder_saved_bytes(const SmkEncoder* h, int B) {
    return h && B > 0 ? h->saved.bytes(B) + smk::ws_round(h->stats_floats * sizeof(float)) : 0;   // stats: train handles only
}

extern "C" int smk_encoder_saved_tensor(const SmkEncoder* h, int B, int i, const char** name, size_t* offset, int* dims) {
    return smk::saved_tensor(h ? &h->saved : nullptr, "smk_encoder_saved_tensor", B, i, name, offset, dims);
}

extern "C" int smk_encoder_forward_saved(const SmkEncoder* h, const float* img, int B, float* pose_cam, float* shape, float* expr,
                                         float* saved, size_t saved_bytes, void* ws, size_t ws_bytes, void* stream) {
    SMK_REQUIRE(h, "smk_encoder_forward_saved: null handle");
    SMK_REQUIRE(B >= 0, "smk_encoder_forward_saved: negative batch");
    if (B == 0) return 0;
    SMK_REQUIRE(img && saved, "smk_encoder_forward_saved: null argument");
    SMK_REQUIRE(saved_bytes > 0 && saved_bytes >= smk_encoder_saved_bytes(h, B), "smk_encoder_forward_saved: saved buffer too small");
    SMK_REQUIRE((pose_cam || !h->present[0]) && (shape || !h->present[1]) && (expr || !h->present[2]),
                "smk_encoder_forward_saved: null output for a backbone this handle holds");
    SMK_REQUIRE(ws && ws_bytes >= smk_encoder_workspace_bytes(h, B), "smk_encoder_forward_saved: workspace too small");
    SMK_REQUIRE(!h->train, "smk_encoder_forward_saved: a train-mode handle runs smk_encoder_forward_train");
    SMK_REQUIRE_WEIGHTS(h, "smk_encoder_forward_saved");
    return encoder_forward(h, img, B, pose_cam, shape, expr, saved, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" size_t smk_encoder_backward_workspace_bytes(const SmkEncoder* h, int B) {
    return h && B > 0 ? 9 * smk::ws_round((size_t)B * h->max_act * sizeof(float)) : 0;     // 3 buffers per backbone
}

extern "C" int smk_encoder_backward(const SmkEncoder* h, int B, const float* saved, size_t saved_bytes, const float* g_pose_cam,
                                    const float* g_shape, const float* g_expr, float* g_img, void* ws, size_t ws_bytes, void* stream) {
    SMK_REQUIRE(h, "smk_encoder_backward: null handle");
    SMK_REQUIRE(B >= 0, "smk_encoder_backward: negative batch");
    if (B == 0) return 0;
    SMK_REQUIRE(saved && g_img, "smk_encoder_backward: null argument");
    SMK_REQUIRE(saved_bytes > 0 && saved_bytes >= smk_encoder_saved_bytes(h, B), "smk_encoder_backward: saved buffer too small");
    SMK_REQUIRE(ws && ws_bytes >= smk_encoder_backward_workspace_bytes(h, B), "smk_encoder_backward: workspace too small");
    SMK_REQUIRE(!h->train, "smk_encoder_backward: a train-mode handle runs smk_encoder_backward_train");
    SMK_REQUIRE_WEIGHTS(h, "smk_encoder_backward");
    cudaStream_t main_st = (cudaStream_t)stream;
    const float* g_out[3] = {g_pose_cam, g_shape, g_expr};
    bool active[3];
    for (int i = 0; i < 3; ++i) active[i] = h->present[i] && g_out[i];          // a NULL upstream gradient launches nothing
    smk::Workspace w(ws, ws_bytes);
    float* bufs[3][3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) bufs[i][j] = w.take<float>((size_t)B * h->max_act);
    SMK_REQUIRE(bufs[2][2] != nullptr, "smk_encoder_backward: workspace carve-up failed");
    auto SV = [&](int i) -> const float* { return saved + (size_t)B * h->saved.off[i]; };
    const bool tc = h->precision >= 1;
    const bool rnd = tc && !h->x3;                  // gradients that feed a TF32 GEMM are rounded (3xTF32 splits them itself)
    const float* g_stem[3] = {nullptr, nullptr, nullptr};
    // the stem dgrad after the join sums every backbone's stem gradient on main_st
    int rc = for_each_unit(h, active, main_st, "smk_encoder_backward", [&](const Unit& unit) {
        const int n = unit.n;
        cudaStream_t st = unit.st;
        int rc = 0;
        const Backbone* bb[2]; float *gy[2], *t1[2], *t2[2];
        for (int k = 0; k < n; ++k) {
            const int i = unit.idx[k];
            bb[k] = &h->bb[i]; gy[k] = bufs[i][0]; t1[k] = bufs[i][1]; t2[k] = bufs[i][2];
        }
        const Backbone& b0b = *bb[0];
        int res = 7;                                 // 224 / 32
        {   // head -> gradient of the cn pre-activation (t1)
            HeadBwd p{};
            int max_out = 0;
            for (int k = 0; k < 2; ++k) {
                const int j = k < n ? k : n - 1;
                const Block& cn = bb[j]->blocks.back();
                p.g[k] = g_out[unit.idx[j]]; p.raw[k] = SV(bb[j]->sv_head); p.codes[k] = bb[j]->codes; p.w[k] = bb[j]->head_w;
                p.cn[k] = SV(cn.sv_a); p.out[k] = t1[j]; p.n_out[k] = bb[j]->n_out;
                max_out = std::max(max_out, bb[j]->n_out);
            }
            const int C = b0b.feat, HW = res * res;
            SMK_TAG("head_dgrad", n * 4.0 * ((double)B * HW * C * 2 + (double)b0b.n_out * C + 2.0 * B * b0b.n_out), n * 2.0 * B * C * b0b.n_out, st);
            SMK_LAUNCH(head_bwd_kernel, dim3(B, smk::cdiv(C, 256), n), dim3(256), (size_t)max_out * 4, st, p, HW, C, rnd ? 1 : 0);
            SMK_CHECK_LAUNCH();
        }
        for (int bi = (int)b0b.blocks.size() - 1; bi >= 0 && !rc; --bi) {
            const Block* b[2] = {&bb[0]->blocks[bi], &bb[n - 1]->blocks[bi]};
            const Block& bk = *b[0];
            // input resolution of the block: the output resolution times the stride, 112 at block 0
            const int ro = res, ri = bi == 0 ? 112 : ro * bk.stride;
            if (bk.kind == CN) {
                const ConvW* c[2] = {&b[0]->pw, &b[1]->pw};
                rc = dgrad_pw(h, n, c, t1, B, ro, ro, nullptr, gy, rnd, tc ? "cn_dgrad_tc" : "cn_dgrad_f32", st);
            } else if (bk.kind == IR) {
                const ConvW* cl[2] = {&b[0]->pwl, &b[1]->pwl};
                const ConvW* cp[2] = {&b[0]->pw, &b[1]->pw};
                const float *dm[2], *am[2];
                for (int k = 0; k < n; ++k) { dm[k] = SV(b[k]->sv_b); am[k] = SV(b[k]->sv_a); }
                rc = dgrad_pw(h, n, cl, gy, B, ro, ro, nullptr, t1, false, tc ? "pwl_dgrad_tc" : "pwl_dgrad_f32", st);
                if (!rc) rc = dgrad_dw(n, b, t1, dm, am, nullptr, B, ri, t2, rnd, st);
                if (!rc) rc = dgrad_pw(h, n, cp, t2, B, ri, ri, bk.skip ? gy : nullptr, t1, rnd, tc ? "pw_dgrad_tc" : "pw_dgrad_f32", st);
                for (int k = 0; k < n; ++k) std::swap(gy[k], t1[k]);
            } else {                                 // DS block 0: the gradient of the stem pre-activation lands in t2
                const ConvW* cp[2] = {&b[0]->pw, &b[1]->pw};
                const float *dm[2], *am[2];
                for (int k = 0; k < n; ++k) { dm[k] = SV(b[k]->sv_a); am[k] = SV(bb[k]->sv_stem); }
                rc = dgrad_pw(h, n, cp, gy, B, ro, ro, nullptr, t1, false, tc ? "ds_pw_dgrad_tc" : "ds_pw_dgrad_f32", st);
                if (!rc) rc = dgrad_dw(n, b, t1, dm, am, bk.skip ? gy : nullptr, B, ri, t2, false, st);
                for (int k = 0; k < n; ++k) g_stem[unit.idx[k]] = t2[k];
            }
            res = ri;
        }
        return rc;
    });
    if (rc) return rc;
    const float* w_stem[3];
    for (int i = 0; i < 3; ++i) w_stem[i] = g_stem[i] ? h->bb[i].stem.dgrad.w : nullptr;
    return enc::stem_dgrad(g_stem, w_stem, B, g_img, main_st);
}

int enc::stem_dgrad(const float* const g[3], const float* const w[3], int B, float* g_img, cudaStream_t st) {
    StemDgrad p{};
    int n_active = 0;
    for (int i = 0; i < 3; ++i) { p.g[i] = g[i]; p.w[i] = g[i] ? w[i] : nullptr; n_active += g[i] != nullptr; }
    const long px = (long)B * 224 * 224;
    SMK_TAG("stem_dgrad", 4.0 * ((double)B * 3 * 224 * 224 + n_active * ((double)B * 112 * 112 * 16 + 27 * 16)), n_active * 2.0 * 27 * 16 * B * 112.0 * 112.0, st);
    SMK_LAUNCH(stem_dgrad_kernel, dim3(smk::cdiv(px, 128)), dim3(128), 0, st, p, B, 224, 224, 112, 112, same_pad_begin(224, 2), g_img);
    SMK_CHECK_LAUNCH();
    return 0;
}
