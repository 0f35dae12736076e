// SmirkEncoder forward: three MobileNetV3-"minimal" backbones + pooled linear heads.
//
// Replaces SmirkEncoder.forward (reference src/smirk_encoder.py:123-133) including the timm backbones
// built at :7-12 (tf_mobilenetv3_small_minimal_100 for pose, ..._large_minimal_100 for shape and
// expression; ReLU only, no squeeze-excite, 3x3 depthwise, BN eps 1e-3, TF-SAME padding) and the
// heads/clamps at :34-45, :66-73, :95-110.  BatchNorm (eval mode) is folded into a per-channel
// scale/bias applied in each convolution's epilogue; activations live in NHWC fp32.
#include "nn_kernels.cuh"
#include "gemm_tc.cuh"
#include "xdw_tc.cuh"
#include <math.h>

namespace {

using smk::TensorCursor;

constexpr float kBnEps = 1e-3f;

struct ConvW { float* w = nullptr; float* wt = nullptr; float* wt_lo = nullptr; float* scale = nullptr; float* bias = nullptr; int cin = 0, cout = 0; };   // w: [K][N] fp32 path, wt: [N][K] tensor-core path (TF32 heads), wt_lo: TF32 tails (3xTF32 path)
enum Kind { DS = 0, IR = 1, CN = 2 };
struct BlockDef { Kind kind; int stride; float exp; int cout; };
struct Block { Kind kind; int stride, cin, mid, cout; bool skip; ConvW pw, dw, pwl; ConvW pw_f32; };   // pw_f32: fp32 [K][N] copy of a DS block's 1x1 (fused stem path)

struct Backbone {
    ConvW stem;
    std::vector<Block> blocks;
    int feat = 0;
    float *head_w = nullptr, *head_b = nullptr;
    int n_out = 0;
    uint8_t* codes = nullptr;
};

const BlockDef kLarge[] = {
    {DS, 1, 1.f, 16},
    {IR, 2, 4.f, 24}, {IR, 1, 3.f, 24},
    {IR, 2, 3.f, 40}, {IR, 1, 3.f, 40}, {IR, 1, 3.f, 40},
    {IR, 2, 6.f, 80}, {IR, 1, 2.5f, 80}, {IR, 1, 2.3f, 80}, {IR, 1, 2.3f, 80},
    {IR, 1, 6.f, 112}, {IR, 1, 6.f, 112},
    {IR, 2, 6.f, 160}, {IR, 1, 6.f, 160}, {IR, 1, 6.f, 160},
    {CN, 1, 1.f, 960}};
const BlockDef kSmall[] = {
    {DS, 2, 1.f, 16},
    {IR, 2, 4.5f, 24}, {IR, 1, 3.67f, 24},
    {IR, 2, 4.f, 40}, {IR, 1, 6.f, 40}, {IR, 1, 6.f, 40},
    {IR, 1, 3.f, 48}, {IR, 1, 3.f, 48},
    {IR, 2, 6.f, 96}, {IR, 1, 6.f, 96}, {IR, 1, 6.f, 96},
    {CN, 1, 1.f, 576}};

int make_divisible(double v, int divisor = 8) {
    int nv = std::max(divisor, (int)(v + divisor / 2.0) / divisor * divisor);
    if (nv < 0.9 * v) nv += divisor;
    return nv;
}

// Consumes (conv weight, bn gamma, beta, mean, var) from the tensor list.
// kind: 0 = 1x1 [Cout,Cin,1,1] -> W[Cin][Cout]; 1 = depthwise [C,1,3,3] -> W[9][C]; 2 = stem [16,3,3,3] -> W[27][16]
bool fold_conv(TensorCursor& cur, int kind, int cin, int cout, bool tc, smk::DeviceArena& arena, ConvW* out, cudaError_t* err, bool x3 = false) {
    const float* w = cur.next(); const float* g = cur.next(); const float* b = cur.next();
    const float* mu = cur.next(); const float* var = cur.next();
    if (!w || !g || !b || !mu || !var) return false;
    std::vector<float> W, Wlo, S(cout), Bi(cout);
    if (kind == 0 && tc) {
        W.resize((size_t)cin * cout);                        // torch layout [Cout][Cin] is already [N][K]
        for (size_t i = 0; i < W.size(); ++i) W[i] = smk::round_tf32_host(w[i]);
        if (x3) {                                            // w = head + tail exactly; the tail is itself a TF32 number up to 2^-22 |w|
            Wlo.resize(W.size());
            for (size_t i = 0; i < W.size(); ++i) Wlo[i] = smk::round_tf32_host(w[i] - W[i]);
        }
    } else if (kind == 0) {
        W.resize((size_t)cin * cout);
        for (int o = 0; o < cout; ++o) for (int c = 0; c < cin; ++c) W[(size_t)c * cout + o] = w[(size_t)o * cin + c];
    } else if (kind == 1) {
        W.resize((size_t)9 * cout);
        for (int c = 0; c < cout; ++c) for (int k = 0; k < 9; ++k) W[(size_t)k * cout + c] = w[(size_t)c * 9 + k];
    } else {
        W.resize((size_t)27 * cout);
        for (int o = 0; o < cout; ++o) for (int k = 0; k < 27; ++k) W[(size_t)k * cout + o] = w[(size_t)o * 27 + k];
    }
    smk::fold_bn(g, b, mu, var, cout, kBnEps, S.data(), Bi.data());
    out->cin = cin; out->cout = cout;
    cudaError_t e = arena.upload(W, (kind == 0 && tc) ? &out->wt : &out->w);
    if (e == cudaSuccess && !Wlo.empty()) e = arena.upload(Wlo, &out->wt_lo);
    if (e == cudaSuccess) e = arena.upload(S, &out->scale);
    if (e == cudaSuccess) e = arena.upload(Bi, &out->bias);
    *err = e;
    return e == cudaSuccess;
}

}  // namespace

struct SmkEncoder {
    Backbone bb[3];
    int n_shape = 300, n_exp = 50, precision = 0;
    size_t max_act = 0;          // floats per image of the largest activation
    bool fuse_xdw = false;       // precision >= 2: inverted-residual blocks use the fused expand+depthwise kernel
    bool x3 = false;             // precision 3: 3xTF32 error-compensated tensor-core arithmetic (fp32-equivalent), no TF32 rounding of activations
    bool present[3] = {false, false, false};   // a handle may hold a subset of the backbones (PoseEncoder / ShapeEncoder / ExpressionEncoder alone)
    smk::DeviceArena arena;
    // Fork/join plumbing for running the backbones as parallel branches of the caller's stream.  A forward takes the
    // next set of a small pool (atomic round-robin), so up to kForkSets forwards of one handle may be in flight on
    // different streams (with distinct workspaces) without sharing an event or a side stream: the handle is re-entrant.
    static constexpr int kForkSets = 8;
    struct ForkSet { cudaStream_t side[2] = {nullptr, nullptr}; cudaEvent_t fork = nullptr, join[2] = {nullptr, nullptr}; };
    ForkSet forks[kForkSets];
    mutable unsigned next_fork = 0;
    ~SmkEncoder() {
        for (auto& f : forks) {
            for (int s = 0; s < 2; ++s) { if (f.side[s]) cudaStreamDestroy(f.side[s]); if (f.join[s]) cudaEventDestroy(f.join[s]); }
            if (f.fork) cudaEventDestroy(f.fork);
        }
    }
};

extern "C" int smk_encoder_create(const SmkEncoderDesc* desc, SmkEncoder** out) {
    SMK_REQUIRE(desc && out, "smk_encoder_create: null argument");
    SMK_REQUIRE(desc->precision >= 0 && desc->precision <= 3,
                "smk_encoder_create: precision must be 0 (fp32 CUDA cores), 1 (tf32 wgmma 1x1 convs), 2 (1 + fused expand/depthwise blocks) or "
                "3 (2 with 3xTF32 error-compensated tensor-core arithmetic: fp32-equivalent results)");
    if (desc->precision >= 1) { if (int rc = smk::tc_init()) return rc; }
    const bool tc = desc->precision >= 1;
    SmkEncoder* h = new SmkEncoder();
    h->n_shape = desc->n_shape; h->n_exp = desc->n_exp; h->precision = tc ? 1 : 0; h->fuse_xdw = desc->precision >= 2; h->x3 = desc->precision == 3;
    const bool x3 = h->x3;
    const int n_outs[3] = {6, desc->n_shape, desc->n_exp + 5};
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 3; ++i) {
        const BlockDef* defs = i == 0 ? kSmall : kLarge;
        const int nb = i == 0 ? (int)(sizeof(kSmall) / sizeof(BlockDef)) : (int)(sizeof(kLarge) / sizeof(BlockDef));
        Backbone& bb = h->bb[i];
        if (desc->n_tensors[i] == 0 || desc->tensors[i] == nullptr) continue;        // backbone not part of this handle
        h->present[i] = true;
        TensorCursor cur{desc->tensors[i], desc->n_tensors[i]};
        bool ok = fold_conv(cur, 2, 3, 16, false, h->arena, &bb.stem, &e);
        int cin = 16, res = 112;
        size_t max_act = (size_t)112 * 112 * 16;
        for (int k = 0; ok && k < nb; ++k) {
            Block b{};
            b.kind = defs[k].kind; b.stride = defs[k].stride; b.cin = cin; b.cout = defs[k].cout;
            b.skip = b.kind != CN && b.stride == 1 && b.cin == b.cout;
            if (b.kind == DS) {
                b.mid = cin;
                ok = fold_conv(cur, 1, cin, cin, false, h->arena, &b.dw, &e);
                if (ok && tc) { TensorCursor again = cur; ok = fold_conv(again, 0, cin, b.cout, false, h->arena, &b.pw_f32, &e); }
                ok = ok && fold_conv(cur, 0, cin, b.cout, tc, h->arena, &b.pw, &e, x3);
            } else if (b.kind == IR) {
                b.mid = make_divisible((double)cin * defs[k].exp);
                ok = fold_conv(cur, 0, cin, b.mid, tc, h->arena, &b.pw, &e, x3) && fold_conv(cur, 1, b.mid, b.mid, false, h->arena, &b.dw, &e) &&
                     fold_conv(cur, 0, b.mid, b.cout, tc, h->arena, &b.pwl, &e, x3);
            } else {
                b.mid = cin;
                ok = fold_conv(cur, 0, cin, b.cout, tc, h->arena, &b.pw, &e, x3);
            }
            max_act = std::max(max_act, (size_t)res * res * b.mid);           // expanded tensor at input resolution
            res = (res + b.stride - 1) / b.stride;
            max_act = std::max(max_act, (size_t)res * res * std::max(b.mid, b.cout));
            cin = b.cout;
            bb.blocks.push_back(b);
        }
        if (!ok || cur.i != cur.n) {
            if (e != cudaSuccess) smk::set_error("smk_encoder_create: upload failed: %s", cudaGetErrorString(e));
            else smk::set_error("smk_encoder_create: backbone %d expects %d tensors (conv weight + 4 BN tensors per conv), got %d",
                                i, cur.i, cur.n);
            delete h; return e != cudaSuccess ? (int)e : -1;
        }
        bb.feat = cin; bb.n_out = n_outs[i];
        h->max_act = std::max(h->max_act, max_act);
        e = h->arena.upload(desc->head_w[i], (size_t)bb.n_out * bb.feat, &bb.head_w);
        if (e == cudaSuccess) e = h->arena.upload(desc->head_b[i], (size_t)bb.n_out, &bb.head_b);
        if (i == 2 && e == cudaSuccess) {                  // smirk_encoder.py:105-108
            std::vector<uint8_t> codes(bb.n_out, 0);
            int ne = desc->n_exp;
            codes[ne] = codes[ne + 1] = 1; codes[ne + 2] = 2; codes[ne + 3] = codes[ne + 4] = 3;
            e = h->arena.upload(codes, &bb.codes);
        }
        if (e != cudaSuccess) { smk::set_error("smk_encoder_create: upload failed: %s", cudaGetErrorString(e)); delete h; return (int)e; }
    }
    if (!h->present[0] && !h->present[1] && !h->present[2]) { smk::set_error("smk_encoder_create: no backbone given"); delete h; return -1; }
    for (auto& f : h->forks) {
        for (int s = 0; s < 2 && e == cudaSuccess; ++s) {
            e = cudaStreamCreateWithFlags(&f.side[s], cudaStreamNonBlocking);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&f.join[s], cudaEventDisableTiming);
        }
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&f.fork, cudaEventDisableTiming);
    }
    if (e != cudaSuccess) { smk::set_error("smk_encoder_create: stream/event creation failed: %s", cudaGetErrorString(e)); delete h; return (int)e; }
    *out = h;
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
        q[k].w = c[k]->w; q[k].wt = c[k]->wt; q[k].wt_lo = c[k]->wt_lo; q[k].scale = c[k]->scale; q[k].bias = c[k]->bias;
        q[k].N = c[k]->cout; q[k].K = c[k]->cin; q[k].mode = 0; q[k].relu = relu ? 1 : 0;
        q[k].res = res ? res[k] : nullptr; q[k].ld_res = c[k]->cout; q[k].out = out[k]; q[k].ld_out = c[k]->cout;
        q[k].round_out = c[k]->wt && !c[k]->wt_lo;      // 3xTF32 consumers split full fp32 activations themselves
    }
    return smk::conv(q[0], st, n == 2 ? &q[1] : nullptr);
}

extern "C" int smk_encoder_forward(const SmkEncoder* h, const float* img, int B, float* pose_cam, float* shape,
                                   float* expr, void* ws, size_t ws_bytes, void* stream) {
    if (B == 0) return 0;                      // empty batch: nothing to do (pointers may be null)
    SMK_REQUIRE(h && img, "smk_encoder_forward: null argument");
    SMK_REQUIRE((pose_cam || !h->present[0]) && (shape || !h->present[1]) && (expr || !h->present[2]),
                "smk_encoder_forward: null output for a backbone this handle holds");
    SMK_REQUIRE(B > 0, "smk_encoder_forward: negative batch");
    SMK_REQUIRE(ws && ws_bytes >= smk_encoder_workspace_bytes(h, B), "smk_encoder_forward: workspace too small");
    cudaStream_t main_st = (cudaStream_t)stream;
    smk::Workspace w(ws, ws_bytes);
    float* bufs[3][4];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 4; ++j) bufs[i][j] = w.take<float>((size_t)B * h->max_act);
    SMK_REQUIRE(bufs[2][3] != nullptr, "smk_encoder_forward: workspace carve-up failed");
    float* outs[3] = {pose_cam, shape, expr};
    // The three backbones are independent (smirk_encoder.py:123-133 merely runs them one after another):
    // fork the two large ones onto the handle's side streams so their many small, latency-bound layers
    // overlap; join before returning.  Event record/wait on other streams is legal under stream capture,
    // so a CUDA graph of the caller's stream gets three parallel branches.
    const int n_present = (int)h->present[0] + (int)h->present[1] + (int)h->present[2];
    const bool concurrent = !smk::profiling() && n_present > 1;   // the event profiler wants one kernel at a time
    const SmkEncoder::ForkSet& fk = h->forks[__atomic_fetch_add(&h->next_fork, 1u, __ATOMIC_RELAXED) % SmkEncoder::kForkSets];
    // precision 2: stem + block 0 (depthwise-separable, 16 channels at 112 x 112) run as one kernel per backbone —
    // the three largest activations never reach HBM.
    const bool fuse_stem = h->fuse_xdw;                           // every backbone starts with a DS block
    if (!fuse_stem && n_present == 3) {   // all three stems in one pass over the image (it is the only tensor the backbones share)
        const float* sw[3]; const float* ss[3]; const float* sb[3]; float* so[3];
        for (int i = 0; i < 3; ++i) { sw[i] = h->bb[i].stem.w; ss[i] = h->bb[i].stem.scale; sb[i] = h->bb[i].stem.bias; so[i] = bufs[i][0]; }
        if (int rc = smk::stem_conv3(img, B, 224, 224, sw, ss, sb, so, main_st)) return rc;
    } else if (!fuse_stem) {
        for (int i = 0; i < 3; ++i)
            if (h->present[i]) { if (int rc = smk::stem_conv(img, B, 224, 224, h->bb[i].stem.w, h->bb[i].stem.scale, h->bb[i].stem.bias, bufs[i][0], main_st)) return rc; }
    }
    if (concurrent) {
        SMK_CHECK_CUDA(cudaEventRecord(fk.fork, main_st));
        for (int s = 0; s < 2; ++s) SMK_CHECK_CUDA(cudaStreamWaitEvent(fk.side[s], fk.fork, 0));
    }
    int rc = 0;                                   // first error; the side streams are joined on every path
    // Work units: the two "large" backbones (shape, expression) have the same layer list, so on the tensor-core path they
    // advance in lock step and every layer of the pair is ONE launch; the small (pose) backbone is its own unit.
    const bool pair = h->precision >= 1 && h->present[1] && h->present[2];
    struct Unit { int n; int idx[2]; cudaStream_t st; };
    Unit units[3]; int n_units = 0;
    if (h->present[0]) units[n_units++] = Unit{1, {0, 0}, main_st};
    if (pair) units[n_units++] = Unit{2, {1, 2}, concurrent ? fk.side[0] : main_st};
    else for (int i = 1; i < 3; ++i) if (h->present[i]) units[n_units++] = Unit{1, {i, i}, concurrent ? fk.side[i - 1] : main_st};
    if (!h->present[0] && n_units > 0) units[0].st = main_st;                        // a lone unit runs on the caller's stream
    for (int u = 0; u < n_units && !rc; ++u) {
        const int n = units[u].n;
        cudaStream_t st = units[u].st;
        const Backbone* bb[2]; float *x[2], *y[2], *e[2], *d[2];
        for (int k = 0; k < n; ++k) {
            const int i = units[u].idx[k];
            bb[k] = &h->bb[i]; x[k] = bufs[i][0]; y[k] = bufs[i][1]; e[k] = bufs[i][2]; d[k] = bufs[i][3];
        }
        int res = 112;
        size_t first = 0;
        if (fuse_stem) {
            const Block& b0 = bb[0]->blocks[0];
            smk::StemDsProblem sp[2];
            for (int k = 0; k < n; ++k) {
                const Block& bk = bb[k]->blocks[0];
                sp[k] = smk::StemDsProblem{bb[k]->stem.w, bb[k]->stem.scale, bb[k]->stem.bias, bk.dw.w, bk.dw.scale, bk.dw.bias,
                                           bk.pw_f32.w, bk.pw_f32.scale, bk.pw_f32.bias, x[k]};
            }
            rc = smk::stem_ds(img, B, 224, 224, sp, n, b0.stride, h->x3 ? 0 : 1, st);
            res = 112 / b0.stride; first = 1;
        }
        for (size_t bi = first; bi < bb[0]->blocks.size() && !rc; ++bi) {
            const Block* b[2] = {&bb[0]->blocks[bi], &bb[n - 1]->blocks[bi]};
            const Block& b0 = *b[0];
            const int ro = (res + b0.stride - 1) / b0.stride;
            const bool rnd = h->precision == 1 && !h->x3;
            const ConvW* pw[2] = {&b[0]->pw, &b[1]->pw};
            const ConvW* pwl[2] = {&b[0]->pwl, &b[1]->pwl};
            if (b0.kind == DS) {
                for (int k = 0; k < n && !rc; ++k)
                    rc = smk::dwconv3x3(x[k], B, res, res, b[k]->cin, b[k]->stride, b[k]->dw.w, b[k]->dw.scale, b[k]->dw.bias, d[k], st, rnd);
                if (!rc) rc = pointwise(n, pw, d, B, ro, ro, false, b0.skip ? x : nullptr, y, st);
            } else if (b0.kind == IR) {
                // The 7x7 layers (a 16x16 window holds 81 useful pixels, 49 outputs) run as 1x1 GEMM + depthwise kernels:
                // most of a window would be halo; every other resolution runs fused.
                constexpr int kXdwMinRes = 8;
                if (h->fuse_xdw && b0.pw.wt && res >= kXdwMinRes) {
                    // expand 1x1 + depthwise 3x3 in one kernel: the expanded tensor never leaves the SM
                    smk::XdwConv q[2];
                    for (int k = 0; k < n; ++k) {
                        q[k] = smk::XdwConv{};
                        q[k].x = x[k]; q[k].B = B; q[k].H = res; q[k].W = res; q[k].Cin = b[k]->cin; q[k].w1t = b[k]->pw.wt; q[k].w1t_lo = b[k]->pw.wt_lo;
                        q[k].scale1 = b[k]->pw.scale; q[k].bias1 = b[k]->pw.bias; q[k].mid = b[k]->mid; q[k].wdw = b[k]->dw.w;
                        q[k].scale2 = b[k]->dw.scale; q[k].bias2 = b[k]->dw.bias; q[k].stride = b[k]->stride; q[k].round_out = h->x3 ? 0 : 1; q[k].out = d[k];
                    }
                    rc = smk::xdw_conv(q[0], st, n == 2 ? &q[1] : nullptr);
                } else {
                    rc = pointwise(n, pw, x, B, res, res, true, nullptr, e, st);
                    for (int k = 0; k < n && !rc; ++k)
                        rc = smk::dwconv3x3(e[k], B, res, res, b[k]->mid, b[k]->stride, b[k]->dw.w, b[k]->dw.scale, b[k]->dw.bias, d[k], st, rnd);
                }
                if (!rc) rc = pointwise(n, pwl, d, B, ro, ro, false, b0.skip ? x : nullptr, y, st);
            } else {
                rc = pointwise(n, pw, x, B, res, res, true, nullptr, y, st);
            }
            if (rc) break;
            for (int k = 0; k < n; ++k) std::swap(x[k], y[k]);
            res = ro;
        }
        if (!rc) {                              // global average pool + head + clamps: one launch per unit
            smk::GapHeadProblem gp[2];
            for (int k = 0; k < n; ++k)
                gp[k] = smk::GapHeadProblem{x[k], bb[k]->head_w, bb[k]->head_b, bb[k]->codes, outs[units[u].idx[k]], bb[k]->n_out};
            rc = smk::gap_head(gp, n, B, res * res, bb[0]->feat, st);
        }
    }
    for (int s = 0; s < 2 && concurrent; ++s) {   // join even after an error so a capturing stream is left consistent
        cudaError_t e1 = cudaEventRecord(fk.join[s], fk.side[s]);
        cudaError_t e2 = e1 == cudaSuccess ? cudaStreamWaitEvent(main_st, fk.join[s], 0) : e1;
        if (!rc && e2 != cudaSuccess) { smk::set_error("smk_encoder_forward: stream join failed: %s", cudaGetErrorString(e2)); rc = (int)e2; }
    }
    return rc;
}
