// Fused "expand 1x1 conv + BN + ReLU  ->  depthwise 3x3 conv + BN + ReLU" for MobileNetV3 inverted-residual
// blocks (reference src/smirk_encoder.py:7-12 -> timm InvertedResidual.conv_pw/bn1/conv_dw/bn2).
//
// The expanded tensor e = ReLU(BN(conv_pw(x))) is the largest activation of every block (4-6x the block's
// input) and in the unfused path is written to HBM by the 1x1 GEMM and read back by the depthwise kernel.
// Here it only ever exists in registers and shared memory:
//
//   CTA = one 16x16-pixel window of e for one image (a 14x14 tile of outputs + halo for stride 1, a 7x7
//         tile for stride 2) x one group of 32-channel chunks of the expanded tensor (the depthwise conv
//         makes channel chunks independent, so low-resolution layers still fill the GPU).  Persistent CTAs;
//         the launcher aims for one per SM, which leaves room on every SM for the other kernels of the
//         concurrent pipeline.
//   producer    one TMA warp: per work item, the whole x window once — two 16x8-pixel boxes per 32-channel
//               k-block (4-D tiled tensor map over NHWC, halo pixels outside the image zero-filled by the hardware)
//               into a window region that stays resident for the item; then only the 1x1 weights (a 32-row box
//               per (chunk, k-block), plus its tails in the 3xTF32 variant) through a small mbarrier ring.
//   MMA         two warpgroups; warpgroup h multiplies window half h (128 pixels x Cin) with wgmma.m64n32k8 TF32
//               (two per k-step, ceil(Cin / 8) k-steps: none over the zero-filled channels past Cin), then
//               (a) accumulator registers -> BN1 + ReLU (+ zero outside the image, which is what the depthwise
//               conv's zero padding of e means) -> shared-memory window E[256][32];
//   depthwise   (b) depthwise 3x3 over E on the CUDA cores (float4 over channels), BN2 + ReLU, optional
//               TF32 rounding, coalesced 256-byte stores of d.
//
// Two schedules.  Serial (xdw_kernel, plain TF32, 288 threads, two CTAs per SM for Cin <= 64): the 8 MMA warps also run
// phase (b), with a CTA barrier after (a) and after (b), so the tensor cores and the FP32 pipes take turns.  Pipelined
// (xdw_ws_kernel, 3xTF32, 512 threads, one CTA per SM): the MMA warpgroups fill a ring of two E slots while a third
// warpgroup runs phase (b) on the slot filled before, so chunk i+1's wgmma and phase (a) overlap chunk i's depthwise
// conv; setmaxnreg gives the MMA warpgroups 168 registers, the depthwise warpgroup 136 and the producer's 40.
// The arithmetic (k-step order, accumulators, BN / ReLU, tap order, rounding) is the same in both, so d and e are too.
//
// Shared memory: [window 0 (, window 1)][weight ring][E slots][parameters][barriers].  The window holds NKB = ceil(Cin / 32)
// k-blocks of 32 KiB (the kernel is instantiated per NKB, Cin <= 160); it is double-buffered where that fits the
// per-SM budget (so the next item's window lands while this item computes), otherwise the producer refills it as soon
// as the item's last chunk has finished its MMAs, during that chunk's phases (a)/(b).  XdwSmem is the plan.
//
// Algorithmic HBM traffic per block drops from  x + 2e + d  to  x + d.  L2 -> shared memory per item: the window
// once (NKB x 32 KiB) + the weights of its chunks (NKB x 4 KiB per chunk, x2 for 3xTF32).
#include "gemm_tc.cuh"
#include "xdw_tc.cuh"
#include "tc_ptx.cuh"

namespace smk {
namespace {

constexpr int BKB = 128, BK = 32, MMA_K = 8;
constexpr int WIN = 16;                         // window edge (pixels of e)
constexpr int HALF_BYTES = 128 * BKB;           // one 16x8-pixel box, 32 channels: 16 KiB
constexpr int KB_BYTES = 2 * HALF_BYTES;        // both halves of the window, one 32-channel k-block: 32 KiB
constexpr int NC = 32;                          // expanded channels per chunk
constexpr int B_BYTES = NC * BKB;               // 4 KiB
constexpr int E_PITCH = NC + 4;                 // floats; 144-byte rows (odd multiple of 16 B): conflict-free 16-byte column writes
constexpr int E_FLOATS = 256 * E_PITCH, E_BYTES = E_FLOATS * 4;    // 36 864 B
constexpr int PAR_ROWS = 13;                     // scale1, bias1, 9 depthwise taps, scale2, bias2
constexpr int PAR_FLOATS = PAR_ROWS * NC, PAR_SLOT_BYTES = PAR_FLOATS * 4;   // one chunk's parameters: 1664 B
constexpr int NUM_WORKERS = 256;                // serial schedule: 8 worker warps; pipelined: the 8 warps of the two MMA warpgroups
constexpr int NUM_THREADS = NUM_WORKERS + 32;   // serial schedule: + the TMA producer warp
// Pipelined schedule: warpgroups 0-1 expand GEMM + phase (a), warpgroup 2 depthwise (one role per thread, cut for 128
// threads), warpgroup 3 the TMA producer (one warp works, three exit).  Every warp starts
// with WS_LAUNCH_REGS; the producer warpgroup gives registers back (setmaxnreg.dec, which may only lower the count) and the
// other three take them (setmaxnreg.inc, which may only raise it).  The budgets fill the 64 K register file exactly.
constexpr int DW_THREADS = 128, WS_THREADS = NUM_WORKERS + DW_THREADS + 128;
constexpr int WS_LAUNCH_REGS = 65536 / WS_THREADS, MMA_REGS = 168, DW_REGS = 136, PROD_REGS = 40;
static_assert(NUM_WORKERS * MMA_REGS + DW_THREADS * DW_REGS + 128 * PROD_REGS == 65536, "register budgets of the pipelined schedule");
static_assert(MMA_REGS >= WS_LAUNCH_REGS && DW_REGS >= WS_LAUNCH_REGS && PROD_REGS <= WS_LAUNCH_REGS,
              "setmaxnreg directions: inc for the MMA and depthwise warpgroups, dec for the producer");
constexpr int MAX_NKB = 5;                      // Cin <= 160
constexpr int SMEM_PER_SM = 228 * 1024, SMEM_PER_CTA = 227 * 1024, SMEM_RESERVED = 1024;   // sm_90 limits

// Shared-memory plan of one window size.  3xTF32 (X3) runs the pipelined schedule, plain TF32 the serial one.
// MINB: resident CTAs per SM the kernel is built for — two for plain TF32 wherever a single window leaves room for them, one for
// 3xTF32 (the pipelined schedule takes the whole register file) and for the deep plain-TF32 windows.
// NE: E slots.  Pipelined: two where they fit beside one window and a 2-stage weight ring, so the MMA warpgroups fill one slot
// while the depthwise warpgroup drains the other; one for NKB = 5 (Cin 160); 2 NE parameter blocks (chunk i's in block
// i % 2NE), so the depthwise warpgroup can stage chunk i + NE's while chunk i's is still in use.  Serial: one E, two parameter
// blocks (chunk parity).
// STAGES: weight stages; NKB where they fit, so the next chunk's weights all load during this chunk's phases (a)/(b).
// WBUF: windows, two where they fit beside MINB CTAs.
template <int NKB, int X3> struct XdwSmem {
    static constexpr int WIN_BYTES = NKB * KB_BYTES;
    static constexpr int STAGE_BYTES = X3 ? 2 * B_BYTES : B_BYTES;      // [w heads] (+ [w tails])
    static constexpr size_t bytes(int wbuf, int stages, int ne) {
        return (size_t)wbuf * WIN_BYTES + stages * STAGE_BYTES + ne * E_BYTES + (X3 ? 2 * ne : 2) * PAR_SLOT_BYTES + 256 + 1024;   // + barriers, alignment slack
    }
    static constexpr bool fits(int wbuf, int stages, int ne, int minb) {
        return bytes(wbuf, stages, ne) <= SMEM_PER_CTA && minb * (bytes(wbuf, stages, ne) + SMEM_RESERVED) <= SMEM_PER_SM;
    }
    static constexpr int MINB = !X3 && fits(1, 2, 1, 2) ? 2 : 1;
    static constexpr int NE = X3 && fits(1, 2, 2, 1) ? 2 : 1;
    static constexpr int STAGES = NKB > 2 && fits(1, NKB, NE, MINB) ? NKB : 2;
    static constexpr int WBUF = fits(2, STAGES, NE, MINB) ? 2 : 1;
    static constexpr size_t SMEM = bytes(WBUF, STAGES, NE);
    static constexpr int RING = WBUF * WIN_BYTES, E_OFF = RING + STAGES * STAGE_BYTES, PAR_OFF = E_OFF + NE * E_BYTES,
                         BAR_OFF = PAR_OFF + (X3 ? 2 * NE : 2) * PAR_SLOT_BYTES;
    static_assert(fits(WBUF, STAGES, NE, MINB), "shared-memory budget");
    static_assert(2 * (STAGES + WBUF + NE) * 8 <= 256, "barrier block");
};
static_assert(XdwSmem<1, 2>::NE == 2 && XdwSmem<2, 2>::NE == 2 && XdwSmem<3, 2>::NE == 2 && XdwSmem<4, 2>::NE == 2,
              "3xTF32: two E slots for every window the encoder launches (Cin <= 112)");

using namespace ptx;                            // PTX wrappers shared by the tensor-core kernels (tc_ptx.cuh)
__device__ __forceinline__ void worker_barrier() { named_barrier(1, NUM_WORKERS); }

struct XdwMaps { CUtensorMap x[2], w[2], wlo[2]; };      // per problem: activations, 1x1 weights (TF32 heads), weight tails

struct XdwArgs {
    int H, W, Ho, Wo;              // e (= x) resolution and output resolution
    int mid, nchunks;              // expanded channels, 32-wide channel chunks
    int groups, chunks_per_group;  // a group owns chunks [g*cpg, min((g+1)*cpg, nchunks)); item = ((img*tiles_y + ty)*tiles_x + tx)*groups + g
    int n_items, B;                // items of the launch (two identically shaped problems may share one, like gemm_tc.cu: image index B.. = problem 1)
    int d_grp, d_tx, d_ty, d_img;  // (group, tile x, tile y, image) digits of the grid size: the item stride of a persistent CTA
    unsigned geom;                 // depthwise row grouping for [columns full|edge][rows full|edge] tiles: byte = rows per thread | row groups << 4
    int pad;                       // TF-SAME pad_begin of the depthwise conv (1 for stride 1, 0 for stride 2 on even sizes)
    int tiles_x, tiles_y;          // output tiles per image
    const float* scale1[2]; const float* bias1[2];  // folded BN of the 1x1 conv        [mid]   (per problem)
    const float* wdw[2];                            // depthwise weights                 [9][mid]
    const float* scale2[2]; const float* bias2[2];  // folded BN of the depthwise conv   [mid]
    float* out[2];                                  // d: [B, Ho, Wo, mid]
    int round_out;
    float* e_out[2];                                // SAVE: e [B, H, W, mid] (per problem)
};

// Persistent CTA: work item = (image, output tile, channel-chunk group), items strided over the grid.  Every role walks the
// same item sequence; the weight ring (and in the pipelined schedule the E ring) runs across item boundaries and the window is
// refilled as soon as it is free, so the loads of item i+1 are in flight while the workers are still busy with item i.
// The item sequence of a CTA advances by gridDim.x; the (group, tile x, tile y, image) digits of the item index are carried
// along incrementally — one runtime decomposition per thread at kernel start instead of four integer divisions per item.
struct Item { int prob, img, oh0, ow0, c_begin, c_end; };
struct ItemIter {
    int item, grp, tx, ty, img2;                // img2: image index over both problems
    __device__ explicit ItemIter(const XdwArgs& a) {
        int v = item = blockIdx.x;
        grp = v % a.groups; v /= a.groups; tx = v % a.tiles_x; v /= a.tiles_x; ty = v % a.tiles_y; img2 = v / a.tiles_y;
    }
    __device__ void next(const XdwArgs& a) {
        item += gridDim.x;
        grp += a.d_grp; if (grp >= a.groups) { grp -= a.groups; ++tx; }
        tx += a.d_tx;   if (tx >= a.tiles_x) { tx -= a.tiles_x; ++ty; }
        ty += a.d_ty;   if (ty >= a.tiles_y) { ty -= a.tiles_y; ++img2; }
        img2 += a.d_img;
    }
    template <int TO> __device__ Item decode(const XdwArgs& a) const {
        Item w;
        w.prob = img2 >= a.B ? 1 : 0; w.img = img2 - w.prob * a.B;
        w.oh0 = ty * TO; w.ow0 = tx * TO;
        w.c_begin = grp * a.chunks_per_group; w.c_end = min(a.nchunks, w.c_begin + a.chunks_per_group);
        return w;
    }
};
// The chunk sequence of a CTA, (problem, chunk) in the order every role walks it (every item has at least one chunk).
template <int TO> struct ChunkIter {
    ItemIter ii;
    int prob, c, c_end;
    __device__ explicit ChunkIter(const XdwArgs& a) : ii(a) { start(a); }
    __device__ bool valid(const XdwArgs& a) const { return ii.item < a.n_items; }
    __device__ void start(const XdwArgs& a) {
        if (valid(a)) { const Item w = ii.decode<TO>(a); prob = w.prob; c = w.c_begin; c_end = w.c_end; }
    }
    __device__ void next(const XdwArgs& a) {
        if (valid(a) && ++c == c_end) { ii.next(a); start(a); }
    }
};

// TMA producer: the x window once per item, then the W1 rows of every (chunk, k-block).
template <int STRIDE, int X3, int NKB>
__device__ __forceinline__ void produce(const XdwMaps& mp, const XdwArgs& a, uint8_t* smem, uint64_t* full, uint64_t* empty,
                                        uint64_t* wfull, uint64_t* wempty) {
    using L = XdwSmem<NKB, X3>;
    constexpr int TO = STRIDE == 1 ? 14 : 7, STAGES = L::STAGES, WBUF = L::WBUF;
    uint8_t* ring = smem + L::RING;
    int it = 0, n = 0;
    for (ItemIter ii(a); ii.item < a.n_items; ii.next(a), ++n) {
        const Item w = ii.decode<TO>(a);
        const int ey0 = w.oh0 * STRIDE - a.pad, ex0 = w.ow0 * STRIDE - a.pad;     // window origin in e / x coordinates
        const int b = n % WBUF;
        mbar_wait(&wempty[b], ((uint32_t)(n / WBUF) & 1u) ^ 1u);
        uint8_t* win = smem + b * L::WIN_BYTES;                                     // [k-block][half][128 pixels][32 channels]
        mbar_expect_tx(&wfull[b], (uint32_t)L::WIN_BYTES);
#pragma unroll
        for (int kb = 0; kb < NKB; ++kb) {
            tma_load_4d(&mp.x[w.prob], win + kb * KB_BYTES, &wfull[b], kb * BK, ex0, ey0, w.img);
            tma_load_4d(&mp.x[w.prob], win + kb * KB_BYTES + HALF_BYTES, &wfull[b], kb * BK, ex0, ey0 + 8, w.img);
        }
        for (int c = w.c_begin; c < w.c_end; ++c)
            for (int kb = 0; kb < NKB; ++kb, ++it) {
                const int s = it % STAGES;
                mbar_wait(&empty[s], ((uint32_t)(it / STAGES) & 1u) ^ 1u);
                uint8_t* st = ring + s * L::STAGE_BYTES;
                mbar_expect_tx(&full[s], (uint32_t)L::STAGE_BYTES);
                tma_load_2d(&mp.w[w.prob], st, &full[s], kb * BK, c * NC);
                if (X3) tma_load_2d(&mp.wlo[w.prob], st + B_BYTES, &full[s], kb * BK, c * NC);
            }
    }
}

// Per-chunk parameters (BN1 scale/bias, nine depthwise taps, BN2 scale/bias: 13 rows of 32 channels) are staged through a
// shared-memory block: thread t < 208 owns one float2 of it, loads it from global memory ahead of time and parks it once the
// block is free, so the global-load latency is off the critical path and phases (a)/(b) read parameters with LDS.  Serial
// schedule: the 256 workers, one chunk ahead, before the MMAs of the previous chunk.  Pipelined: the 128 depthwise threads
// (two float2 each for the first 80), NE chunks ahead, during a depthwise conv.  Channels past `mid` get zero scale and bias.
struct ParLoader {
    const float* src[2];
    int prow, pcol;
    bool owner;
    __device__ ParLoader(const XdwArgs& a, int t) : src{nullptr, nullptr}, prow(t >> 4), pcol((t & 15) * 2), owner(t < PAR_ROWS * 16) {
        if (owner) {
#pragma unroll
            for (int q = 0; q < 2; ++q)
                src[q] = (prow == 0 ? a.scale1[q] : prow == 1 ? a.bias1[q] : prow == 11 ? a.scale2[q] : prow == 12 ? a.bias2[q]
                                                                                  : a.wdw[q] + (size_t)(prow - 2) * a.mid) + pcol;
        }
    }
    // SELECT: pick the problem's pointer with a select rather than an index, which keeps src out of local memory in the
    // pipelined kernel's depthwise warpgroup; the serial kernel's 96-register allocation spills less with the index.
    template <bool SELECT = false> __device__ float2 load(const XdwArgs& a, int prob, int c) const {
        float2 v = make_float2(0.f, 0.f);
        if (owner && c * NC + pcol < a.mid) v = __ldg(reinterpret_cast<const float2*>((SELECT ? (prob ? src[1] : src[0]) : src[prob]) + c * NC));
        return v;
    }
    __device__ void park(float* par, const float2& v) const {
        if (owner) *reinterpret_cast<float2*>(par + prow * NC + pcol) = v;
    }
};

// Expand GEMM of one chunk: rows [64 mb, 64 mb + 64) of this warpgroup's window half x the chunk's 32 weight rows, over the
// NKB k-blocks of weights streamed through the ring (k-block `it` in stage it % STAGES).
template <int X3, int NKB, int KSL>
__device__ __forceinline__ void expand_gemm(float (&acc)[2][NC / 2], const uint8_t* win, uint8_t* ring, uint64_t* full, uint64_t* empty,
                                            int& it, int wq, int lane) {
    using L = XdwSmem<NKB, X3>;
    constexpr int STAGES = L::STAGES;
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int i = 0; i < NC / 2; ++i) acc[mb][i] = 0.f;
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb, ++it) {
        // k-steps of this k-block: all four, except KSL in the last one, where the steps over the channels past Cin
        // (zero-filled by TMA) would only add zeros.  Known at compile time, so no wgmma sits behind a branch.
        const int nks = kb + 1 < NKB ? BK / MMA_K : KSL;
        const int s = it % STAGES;
        mbar_wait(&full[s], (uint32_t)(it / STAGES) & 1u);
        const uint8_t* xa = win + kb * KB_BYTES;
        const uint32_t sb = smem_u32(ring + s * L::STAGE_BYTES);
        if constexpr (X3 != 0) {
            uint32_t hi[2][BK / MMA_K][4], lo[2][BK / MMA_K][4];
#pragma unroll
            for (int mb = 0; mb < 2; ++mb)
#pragma unroll
                for (int k = 0; k < nks; ++k) {
                    float v[4];
                    load_a_frag(xa, mb * 64, k * MMA_K, wq, lane, v);
                    split_frag(v, hi[mb][k], lo[mb][k]);
                }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < nks; ++k) {
                const uint64_t db = make_smem_desc(sb + k * MMA_K * 4);
                const uint64_t dbl = make_smem_desc(sb + B_BYTES + k * MMA_K * 4);
#pragma unroll
                for (int mb = 0; mb < 2; ++mb) {
                    Wgmma<NC>::rs(acc[mb], hi[mb][k], db, 1u);       // x_hi * w_hi
                    Wgmma<NC>::rs(acc[mb], lo[mb][k], db, 1u);       // x_lo * w_hi
                    Wgmma<NC>::rs(acc[mb], hi[mb][k], dbl, 1u);      // x_hi * w_lo
                }
            }
        } else {
            const uint32_t sa = smem_u32(xa);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < nks; ++k) {
                const uint64_t db = make_smem_desc(sb + k * MMA_K * 4);
#pragma unroll
                for (int mb = 0; mb < 2; ++mb)
                    Wgmma<NC>::ss(acc[mb], make_smem_desc(sa + mb * 64 * BKB + k * MMA_K * 4), db, 1u);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        mbar_arrive_if(&empty[s], lane == 0);
    }
}

// Phase (a): accumulators -> BN1 + ReLU -> E.  Channels past `mid` have zero scale and bias in the parameter block, pixels
// outside the image are zeroed: that is the zero padding of e the depthwise conv expects.  SAVE: also store e for the pixels
// the item owns.
template <int STRIDE, bool SAVE>
__device__ __forceinline__ void bn1_relu(const float (&acc)[2][NC / 2], float* E, const float* par, const XdwArgs& a, const Item& w,
                                         int ch0, int half, int wq, int lane) {
    constexpr int TO = STRIDE == 1 ? 14 : 7;
    const int ey0 = w.oh0 * STRIDE - a.pad, ex0 = w.ow0 * STRIDE - a.pad;
#pragma unroll
    for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int r = mb * 64 + wq * 16 + (lane >> 2) + 8 * hr;      // row within the half: r = hh*16 + ww
            const int ey = ey0 + half * 8 + (r >> 4), ex = ex0 + (r & 15);
            const bool inside = ey >= 0 && ey < a.H && ex >= 0 && ex < a.W;
            float* erow = E + (size_t)(half * 128 + r) * E_PITCH;
            bool own = false;
            float* esave = nullptr;
            if constexpr (SAVE) {
                own = inside && ey >= w.oh0 * STRIDE && ey < (w.oh0 + TO) * STRIDE && ex >= w.ow0 * STRIDE && ex < (w.ow0 + TO) * STRIDE;
                esave = a.e_out[w.prob] + (((size_t)w.img * a.H + ey) * a.W + ex) * a.mid + ch0;
            }
#pragma unroll
            for (int j = 0; j < NC / 8; ++j) {
                const int ch = 8 * j + 2 * (lane & 3);
                float2 o = make_float2(0.f, 0.f);
                if (inside) {
                    const float2 sc = *reinterpret_cast<const float2*>(par + ch);
                    const float2 bi = *reinterpret_cast<const float2*>(par + NC + ch);
                    o.x = fmaxf(fmaf(acc[mb][4 * j + 2 * hr], sc.x, bi.x), 0.f);
                    o.y = fmaxf(fmaf(acc[mb][4 * j + 2 * hr + 1], sc.y, bi.y), 0.f);
                }
                *reinterpret_cast<float2*>(erow + ch) = o;
                if (SAVE && own && ch0 + ch < a.mid) *reinterpret_cast<float2*>(esave + ch) = o;
            }
        }
}

// Depthwise role: a run of DWC adjacent output columns starting at ox (dw_cols: two in the pipelined schedule at stride 1,
// else one), and row group rg, of one channel quad.  The tile's column runs x as many row groups as fit in the schedule's
// slots (depthwise threads / 8 channel quads: 32 serial, 16 pipelined), so every slot gets about the same number of outputs.
// A tile has TO columns / rows except in the last tile column / row: the role for both column counts is worked out once
// (bytes: ox full, rg full, ox edge, rg edge), the row grouping of the four tile kinds comes from the host (a.geom); the item
// loop only selects (dw_rows).
__host__ __device__ constexpr int dw_cols(int stride, bool pipelined) { return stride == 1 && pipelined ? 2 : 1; }
template <int STRIDE, int DWC> __device__ __forceinline__ unsigned dw_role(const XdwArgs& a, int slot) {
    constexpr int TO = STRIDE == 1 ? 14 : 7, NCR = (TO + DWC - 1) / DWC;
    const int ncr_e = (a.Wo - (a.tiles_x - 1) * TO + DWC - 1) / DWC;   // column runs of an edge tile
    return (unsigned)(slot % NCR * DWC) | (unsigned)(slot / NCR) << 8 | (unsigned)(slot % ncr_e * DWC) << 16 | (unsigned)(slot / ncr_e) << 24;
}
struct DwRows { int ox, ncol, oy0, oy1; };      // output columns [ox, ox + ncol) and output rows [oy0, oy1) of the tile
template <int STRIDE, int DWC> __device__ __forceinline__ DwRows dw_rows(const XdwArgs& a, const ItemIter& ii, unsigned role) {
    constexpr int TO = STRIDE == 1 ? 14 : 7;
    const bool col_e = ii.tx == a.tiles_x - 1, row_e = ii.ty == a.tiles_y - 1;
    const int nrows = row_e ? a.Ho - (a.tiles_y - 1) * TO : TO, ncols = col_e ? a.Wo - (a.tiles_x - 1) * TO : TO;
    const unsigned g8 = a.geom >> ((col_e ? 16 : 0) + (row_e ? 8 : 0));
    const int rpt = (int)(g8 & 15u), n_rg = (int)((g8 >> 4) & 15u);
    const unsigned r16 = role >> (col_e ? 16 : 0);
    const int rg = (int)((r16 >> 8) & 255u);
    DwRows d;
    d.ox = (int)(r16 & 255u); d.ncol = min(DWC, ncols - d.ox);
    d.oy0 = rg * rpt; d.oy1 = rg < n_rg ? min(nrows, d.oy0 + rpt) : 0;
    return d;
}

// Phase (b): depthwise 3x3 over E, BN2 + ReLU, optional TF32 rounding, store of d.  Tap order per output stays (ky, kx)
// ascending, one fmaf chain from zero -> same rounding as the unfused path.
// Stride 1: one thread owns DWC adjacent output columns of one channel quad and walks down their rows; every E row it reads
// feeds those columns and the up to three output rows that use it, through rolling accumulators.
//   DWC = 1 (serial schedule): 3 LDS.128 per input row; the accumulators of the two rows above oy0 are computed and dropped,
//     which keeps the loop within the 96 registers of the two-CTA serial kernel.
//   DWC = 2 (pipelined schedule): 4 LDS.128 per input row for both columns; p = output r-2 (gets its ky=2 taps from row r,
//     then is stored), q = output r-1 (ky=1, then becomes p), and a fresh one for output r (ky=0, then becomes q).  The first
//     two and the last two input rows are peeled, so no accumulator is started for an output outside [oy0, oy1).  A run cut
//     short by the tile edge (ncol = 1) still computes its second column, which lies inside the 16-pixel window, and does
//     not store it.
// Stride 2: one thread owns one output column; a row of E is shared by two output rows at most.
template <int STRIDE, int DWC>
__device__ __forceinline__ void depthwise(const float* E, const float* par, const XdwArgs& a, const Item& w, int ch0, int cq, const DwRows& rows) {
    static_assert(STRIDE == 1 || DWC == 1, "stride 2 runs one column per role");
    if (cq * 4 < a.mid - ch0 && rows.oy0 < rows.oy1) {
        const int ch = ch0 + cq * 4;
        float4 k[9];
#pragma unroll
        for (int q = 0; q < 9; ++q) k[q] = *reinterpret_cast<const float4*>(par + (2 + q) * NC + cq * 4);
        const float4 s2 = *reinterpret_cast<const float4*>(par + 11 * NC + cq * 4);
        const float4 b2 = *reinterpret_cast<const float4*>(par + 12 * NC + cq * 4);
        float* orow = a.out[w.prob] + (((size_t)w.img * a.Ho + w.oh0 + rows.oy0) * a.Wo + w.ow0 + rows.ox) * a.mid + ch;
        const size_t orow_stride = (size_t)a.Wo * a.mid;
        auto bn2 = [&](const float4& acc4) {
            float4 o = fma4(acc4, s2, b2);
            o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f);
            if (a.round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
            return o;
        };
        auto emit = [&](const float4& acc4) {
            *reinterpret_cast<float4*>(orow) = bn2(acc4);
            orow += orow_stride;
        };
        const float* e = E + (size_t)((rows.oy0 * STRIDE) * WIN + rows.ox * STRIDE) * E_PITCH + cq * 4;
        const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
        if (STRIDE == 1 && DWC == 1) {
            float4 acc0 = zero, acc1 = zero, acc2 = zero;          // outputs r-2 (gets ky=2), r-1 (ky=1), r (ky=0)
            const int n_in = rows.oy1 - rows.oy0 + 2;
#pragma unroll 3
            for (int r = 0; r < n_in; ++r, e += WIN * E_PITCH) {
                const float4 x0 = *reinterpret_cast<const float4*>(e);
                const float4 x1 = *reinterpret_cast<const float4*>(e + E_PITCH);
                const float4 x2 = *reinterpret_cast<const float4*>(e + 2 * E_PITCH);
                fma4_acc(acc0, x0, k[6]); fma4_acc(acc0, x1, k[7]); fma4_acc(acc0, x2, k[8]);
                fma4_acc(acc1, x0, k[3]); fma4_acc(acc1, x1, k[4]); fma4_acc(acc1, x2, k[5]);
                fma4_acc(acc2, x0, k[0]); fma4_acc(acc2, x1, k[1]); fma4_acc(acc2, x2, k[2]);
                if (r >= 2) emit(acc0);
                acc0 = acc1; acc1 = acc2; acc2 = zero;
            }
        } else if (STRIDE == 1) {
            struct Acc { float4 c[DWC]; };             // the DWC columns of one output row
            float4 x[DWC + 2];
            auto load = [&](int r) {
#pragma unroll
                for (int j = 0; j < DWC + 2; ++j) x[j] = *reinterpret_cast<const float4*>(e + (r * WIN + j) * E_PITCH);
            };
            auto fresh = [&]() {
                Acc acc;
#pragma unroll
                for (int j = 0; j < DWC; ++j) acc.c[j] = zero;
                return acc;
            };
            auto taps = [&](Acc& acc, int ky) {    // acc += the ky row of taps over the loaded E row, every column
#pragma unroll
                for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                    for (int j = 0; j < DWC; ++j) fma4_acc(acc.c[j], x[kx + j], k[3 * ky + kx]);
            };
            auto store = [&](const Acc& acc) {
#pragma unroll
                for (int j = 0; j < DWC; ++j)
                    if (j == 0 || j < rows.ncol) *reinterpret_cast<float4*>(orow + j * a.mid) = bn2(acc.c[j]);
                orow += orow_stride;
            };
            const int n_out = rows.oy1 - rows.oy0;
            Acc p, q = fresh();
            load(0); taps(q, 0);                                            // output 0: ky=0
            load(1); p = q; taps(p, 1);                                     // output 0: ky=1
            if (n_out > 1) { q = fresh(); taps(q, 0); }                     // output 1: ky=0
#pragma unroll 2
            for (int r = 2; r < n_out; ++r) {                               // outputs r-2 (done), r-1, r
                load(r);
                taps(p, 2); store(p);
                p = q; taps(p, 1);
                q = fresh(); taps(q, 0);
            }
            if (n_out > 1) { load(n_out); taps(p, 2); store(p); p = q; taps(p, 1); }
            load(n_out + 1); taps(p, 2); store(p);                          // the last output: ky=2
        } else {
            float4 p0 = *reinterpret_cast<const float4*>(e);
            float4 p1 = *reinterpret_cast<const float4*>(e + E_PITCH);
            float4 p2 = *reinterpret_cast<const float4*>(e + 2 * E_PITCH);
            for (int oy = rows.oy0; oy < rows.oy1; ++oy) {
                e += WIN * E_PITCH;
                float4 acc4 = zero;
                fma4_acc(acc4, p0, k[0]); fma4_acc(acc4, p1, k[1]); fma4_acc(acc4, p2, k[2]);
                const float4 m0 = *reinterpret_cast<const float4*>(e);
                const float4 m1 = *reinterpret_cast<const float4*>(e + E_PITCH);
                const float4 m2 = *reinterpret_cast<const float4*>(e + 2 * E_PITCH);
                fma4_acc(acc4, m0, k[3]); fma4_acc(acc4, m1, k[4]); fma4_acc(acc4, m2, k[5]);
                e += WIN * E_PITCH;
                p0 = *reinterpret_cast<const float4*>(e);
                p1 = *reinterpret_cast<const float4*>(e + E_PITCH);
                p2 = *reinterpret_cast<const float4*>(e + 2 * E_PITCH);
                fma4_acc(acc4, p0, k[6]); fma4_acc(acc4, p1, k[7]); fma4_acc(acc4, p2, k[8]);
                emit(acc4);
            }
        }
    }
}

// Shared-memory pointers of one CTA: [window 0 (, window 1)][weight ring][E slots][parameter blocks][barriers].
template <int NKB, int X3> struct XdwShared {
    using L = XdwSmem<NKB, X3>;
    uint8_t* smem;
    float* E;                   // [NE][256][E_PITCH]
    float* PAR;                 // [X3 ? 2 NE : 2][PAR_ROWS][NC]
    uint64_t *full, *empty;     // weight stage s loaded / free
    uint64_t *wfull, *wempty;   // window b loaded (TMA transaction count) / free: its item's last chunk has finished its MMAs
    uint64_t *efull, *eempty;   // pipelined: E slot s written by phase (a) / drained by phase (b)
    __device__ explicit XdwShared(uint8_t* raw) {
        // 1024-byte alignment for SWIZZLE_128B; offset arithmetic (not an integer round-trip of the pointer) keeps the shared
        // address space visible to the compiler, so E is accessed with LDS/STS instead of generic LD/ST.
        smem = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
        E = reinterpret_cast<float*>(smem + L::E_OFF);
        PAR = reinterpret_cast<float*>(smem + L::PAR_OFF);
        full = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
        empty = full + L::STAGES;
        wfull = empty + L::STAGES;
        wempty = wfull + L::WBUF;
        efull = wempty + L::WBUF;
        eempty = efull + L::NE;
    }
};

// Serial schedule (plain TF32).  For each chunk all 8 worker warps run the expand MMAs, phase (a) into E, a barrier, phase
// (b) from E, a barrier.  X3 != 0: see xdw_ws_kernel.
template <int STRIDE, int X3, int NKB, int KSL, bool SAVE>
__global__ void __launch_bounds__(NUM_THREADS, XdwSmem<NKB, X3>::MINB)
xdw_kernel(const __grid_constant__ XdwMaps mp, const XdwArgs a) {
    using L = XdwSmem<NKB, X3>;
    constexpr int TO = STRIDE == 1 ? 14 : 7;
    extern __shared__ uint8_t smem_raw[];
    const XdwShared<NKB, X3> sh(smem_raw);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == NUM_WORKERS / 32 && lane == 0) {
        prefetch_tensormap(&mp.x[0]);
        prefetch_tensormap(&mp.w[0]);
        for (int s = 0; s < L::STAGES; ++s) { mbar_init(&sh.full[s], 1); mbar_init(&sh.empty[s], NUM_WORKERS / 32); }
        for (int b = 0; b < L::WBUF; ++b) { mbar_init(&sh.wfull[b], 1); mbar_init(&sh.wempty[b], NUM_WORKERS / 32); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == NUM_WORKERS / 32) {
        if (lane == 0) produce<STRIDE, X3, NKB>(mp, a, sh.smem, sh.full, sh.empty, sh.wfull, sh.wempty);
        return;
    }

    // ===== workers: 8 warps =====
    const int half = warp >> 2, wq = warp & 3;         // warpgroup = window half (rows 128 half ..), warp within it
    const int t = threadIdx.x;                         // 0..255
    const int cq = t & 7;                              // depthwise role: channel quad within the chunk, output slot t >> 3
    // Parameters of chunk i+1 are loaded before the MMAs of chunk i and parked (slot (i+1) & 1) after its phase (a).
    const ParLoader pl(a, t);
    ItemIter ii(a);
    if (ii.item < a.n_items) { const Item w0 = ii.decode<TO>(a); pl.park(sh.PAR, pl.load(a, w0.prob, w0.c_begin)); }
    worker_barrier();
    constexpr int DWC = dw_cols(STRIDE, false);
    const unsigned role = dw_role<STRIDE, DWC>(a, t >> 3);
    int cc = 0, it = 0;
    for (int n = 0; ii.item < a.n_items; ++n) {
      const Item w = ii.decode<TO>(a);
      const int wb = n % L::WBUF;
      const uint8_t* win = sh.smem + wb * L::WIN_BYTES + half * HALF_BYTES;     // this warpgroup's half of k-block 0
      mbar_wait(&sh.wfull[wb], (uint32_t)(n / L::WBUF) & 1u);
      const DwRows rows = dw_rows<STRIDE, DWC>(a, ii, role);
      int next_first = -1, next_prob = 0;              // first chunk (and problem) of this CTA's next item (-1: none)
      ii.next(a);
      if (ii.item < a.n_items) { const Item wn = ii.decode<TO>(a); next_first = wn.c_begin; next_prob = wn.prob; }
      for (int c = w.c_begin; c < w.c_end; ++c, ++cc) {
        const int buf = cc & 1;
        const float* par = sh.PAR + buf * PAR_FLOATS;
        const int c_next = c + 1 < w.c_end ? c + 1 : next_first;
        float2 pf = make_float2(0.f, 0.f);
        if (c_next >= 0) pf = pl.load(a, c + 1 < w.c_end ? w.prob : next_prob, c_next);
        float acc[2][NC / 2];
        expand_gemm<X3, NKB, KSL>(acc, win, sh.smem + L::RING, sh.full, sh.empty, it, wq, lane);
        mbar_arrive_if(&sh.wempty[wb], lane == 0 && c + 1 == w.c_end);     // the item's last MMAs have read the window
        bn1_relu<STRIDE, SAVE>(acc, sh.E, par, a, w, c * NC, half, wq, lane);
        if (c_next >= 0) pl.park(sh.PAR + (buf ^ 1) * PAR_FLOATS, pf);     // slot buf^1 was last read in the previous chunk's phase (b)
        worker_barrier();
        depthwise<STRIDE, DWC>(sh.E, par, a, w, c * NC, cq, rows);
        worker_barrier();                              // E and the parameter slot are free for the next chunk
      }
    }
}

// Pipelined, warp-specialized schedule (3xTF32).  The MMA warpgroups run chunk i's expand GEMM and phase (a) into E slot
// i % NE, hand the slot to the depthwise warpgroup and go straight on to chunk i+1, so the tensor cores work on one chunk
// while the FP32 pipes run the depthwise conv of the previous one.  Slot hand-offs are mbarriers (efull: 256 MMA-thread
// arrivals, eempty: 128 depthwise-thread arrivals).  The depthwise warpgroup, which has slack on most layer shapes, also
// stages the parameter blocks, so an eempty phase means "slot free and the next chunk's parameters in place" and the MMA
// warpgroups go from their GEMM to phase (a) without a barrier between them.  No CTA-wide barrier inside the item loop; the E
// ring runs across item boundaries like the weight ring.
template <int STRIDE, int X3, int NKB, int KSL, bool SAVE>
__global__ void __launch_bounds__(WS_THREADS, 1)
xdw_ws_kernel(const __grid_constant__ XdwMaps mp, const XdwArgs a) {
    using L = XdwSmem<NKB, X3>;
    constexpr int TO = STRIDE == 1 ? 14 : 7, NE = L::NE;
    constexpr int PROD_WARP = (NUM_WORKERS + DW_THREADS) / 32;
    extern __shared__ uint8_t smem_raw[];
    const XdwShared<NKB, X3> sh(smem_raw);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == PROD_WARP && lane == 0) {
        prefetch_tensormap(&mp.x[0]);
        prefetch_tensormap(&mp.w[0]);
        prefetch_tensormap(&mp.wlo[0]);
        for (int s = 0; s < L::STAGES; ++s) { mbar_init(&sh.full[s], 1); mbar_init(&sh.empty[s], NUM_WORKERS / 32); }
        for (int b = 0; b < L::WBUF; ++b) { mbar_init(&sh.wfull[b], 1); mbar_init(&sh.wempty[b], NUM_WORKERS / 32); }
        for (int s = 0; s < NE; ++s) { mbar_init(&sh.efull[s], NUM_WORKERS); mbar_init(&sh.eempty[s], DW_THREADS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp >= PROD_WARP) {                           // warpgroup 3: the TMA producer
        setmaxnreg_dec<PROD_REGS>();
        if (warp == PROD_WARP && lane == 0) produce<STRIDE, X3, NKB>(mp, a, sh.smem, sh.full, sh.empty, sh.wfull, sh.wempty);
        return;
    }

    if (warp >= NUM_WORKERS / 32) {                    // warpgroup 2: phase (b) of every chunk, slot by slot
        setmaxnreg_inc<DW_REGS>();
        const int d = threadIdx.x - NUM_WORKERS, cq = d & 7;
        constexpr int DWC = dw_cols(STRIDE, true);
        const unsigned role = dw_role<STRIDE, DWC>(a, d >> 3);
        // The parameter block of chunk i + NE is staged here: its global loads are issued before chunk i's depthwise conv and
        // parked after it, then the eempty arrival publishes slot and block together.  Block (i + NE) % (2 NE) was last read
        // by chunk i - NE, whose phase (a) and (b) are complete for every thread once chunk i's efull has completed.
        const ParLoader pl0(a, d), pl1(a, d + DW_THREADS);               // float2 owners d and d + 128 of the 208
        ChunkIter<TO> ahead(a);
        for (int j = 0; j < NE; ++j, ahead.next(a)) {                     // blocks of the first NE chunks, then free slots
            if (ahead.valid(a)) {
                float* par = sh.PAR + j * PAR_FLOATS;
                pl0.park(par, pl0.load<true>(a, ahead.prob, ahead.c)); pl1.park(par, pl1.load<true>(a, ahead.prob, ahead.c));
            }
            mbar_arrive(&sh.eempty[j]);
        }
        int cc = 0;
        for (ItemIter ii(a); ii.item < a.n_items; ii.next(a)) {
            const Item w = ii.decode<TO>(a);
            const DwRows rows = dw_rows<STRIDE, DWC>(a, ii, role);
            for (int c = w.c_begin; c < w.c_end; ++c, ++cc, ahead.next(a)) {
                const int s = cc % NE;
                const bool stage = ahead.valid(a);
                float2 pf0 = make_float2(0.f, 0.f), pf1 = pf0;
                if (stage) { pf0 = pl0.load<true>(a, ahead.prob, ahead.c); pf1 = pl1.load<true>(a, ahead.prob, ahead.c); }
                mbar_wait(&sh.efull[s], (uint32_t)(cc / NE) & 1u);
                depthwise<STRIDE, DWC>(sh.E + s * E_FLOATS, sh.PAR + (cc % (2 * NE)) * PAR_FLOATS, a, w, c * NC, cq, rows);
                if (stage) {
                    float* par = sh.PAR + ((cc + NE) % (2 * NE)) * PAR_FLOATS;
                    pl0.park(par, pf0); pl1.park(par, pf1);
                }
                mbar_arrive(&sh.eempty[s]);            // slot s drained, chunk cc + NE's parameters staged
            }
        }
        return;
    }

    // warpgroups 0-1: expand GEMM of window half `half`, then phase (a) into the next free E slot.  The two warpgroups
    // share no barrier in the loop: each waits for its weights, its window and the E slot on its own.
    setmaxnreg_inc<MMA_REGS>();
    const int half = warp >> 2, wq = warp & 3;
    int cc = 0, it = 0, n = 0;
    for (ItemIter ii(a); ii.item < a.n_items; ii.next(a), ++n) {
        const Item w = ii.decode<TO>(a);
        const int wb = n % L::WBUF;
        const uint8_t* win = sh.smem + wb * L::WIN_BYTES + half * HALF_BYTES;
        mbar_wait(&sh.wfull[wb], (uint32_t)(n / L::WBUF) & 1u);
        for (int c = w.c_begin; c < w.c_end; ++c, ++cc) {
            const int s = cc % NE;
            float acc[2][NC / 2];
            expand_gemm<X3, NKB, KSL>(acc, win, sh.smem + L::RING, sh.full, sh.empty, it, wq, lane);
            mbar_arrive_if(&sh.wempty[wb], lane == 0 && c + 1 == w.c_end);
            mbar_wait(&sh.eempty[s], (uint32_t)(cc / NE) & 1u);     // slot drained by chunk cc - NE, chunk cc's parameters staged
            bn1_relu<STRIDE, SAVE>(acc, sh.E + s * E_FLOATS, sh.PAR + (cc % (2 * NE)) * PAR_FLOATS, a, w, c * NC, half, wq, lane);
            mbar_arrive(&sh.efull[s]);
        }
    }
}

template <int STRIDE, int X3, int NKB, int KSL, bool SAVE>
int launch(const XdwMaps& mp, const XdwArgs& a, int grid, cudaStream_t st) {
    constexpr size_t smem = XdwSmem<NKB, X3>::SMEM;
    if constexpr (X3 != 0) {
        SMK_CHECK_CUDA((set_max_dynamic_smem<xdw_ws_kernel<STRIDE, X3, NKB, KSL, SAVE>>((int)smem)));
        SMK_LAUNCH((xdw_ws_kernel<STRIDE, X3, NKB, KSL, SAVE>), dim3(grid), dim3(WS_THREADS), smem, st, mp, a);
    } else {
        SMK_CHECK_CUDA((set_max_dynamic_smem<xdw_kernel<STRIDE, X3, NKB, KSL, SAVE>>((int)smem)));
        SMK_LAUNCH((xdw_kernel<STRIDE, X3, NKB, KSL, SAVE>), dim3(grid), dim3(NUM_THREADS), smem, st, mp, a);
    }
    SMK_CHECK_LAUNCH();
    return 0;
}

template <int STRIDE, int X3, int NKB, int KSL>
int launch_save(const XdwMaps& mp, const XdwArgs& a, int grid, cudaStream_t st) {
    return a.e_out[0] ? launch<STRIDE, X3, NKB, KSL, true>(mp, a, grid, st) : launch<STRIDE, X3, NKB, KSL, false>(mp, a, grid, st);
}

template <int STRIDE, int X3, int NKB>
int launch_ksl(int ksl, const XdwMaps& mp, const XdwArgs& a, int grid, cudaStream_t st) {
    switch (ksl) {
        case 1: return launch_save<STRIDE, X3, NKB, 1>(mp, a, grid, st);
        case 2: return launch_save<STRIDE, X3, NKB, 2>(mp, a, grid, st);
        case 3: return launch_save<STRIDE, X3, NKB, 3>(mp, a, grid, st);
        default: return launch_save<STRIDE, X3, NKB, 4>(mp, a, grid, st);
    }
}

// instantiation by window size: Cin = 32 (nkb - 1) + 8 ksl (rounded up to a multiple of 8), nkb <= MAX_NKB
template <int STRIDE, int X3>
int launch_cin(int Cin, const XdwMaps& mp, const XdwArgs& a, int grid, cudaStream_t st) {
    static_assert(MAX_NKB == 5, "one case per window size");
    const int nkb = cdiv(Cin, BK), ksl = cdiv(Cin, MMA_K) - (nkb - 1) * (BK / MMA_K);
    switch (nkb) {
        case 1: return launch_ksl<STRIDE, X3, 1>(ksl, mp, a, grid, st);
        case 2: return launch_ksl<STRIDE, X3, 2>(ksl, mp, a, grid, st);
        case 3: return launch_ksl<STRIDE, X3, 3>(ksl, mp, a, grid, st);
        case 4: return launch_ksl<STRIDE, X3, 4>(ksl, mp, a, grid, st);
        default: return launch_ksl<STRIDE, X3, 5>(ksl, mp, a, grid, st);
    }
}

}  // namespace

int xdw_conv(const XdwConv& p, cudaStream_t st, const XdwConv* p2) {
    const int nprob = p2 ? 2 : 1;
    SMK_REQUIRE(p.stride == 1 || p.stride == 2, "xdw_conv: stride must be 1 or 2");
    SMK_REQUIRE(p.Cin % 4 == 0 && p.mid % 4 == 0, "xdw_conv: Cin and mid must be multiples of 4");
    SMK_REQUIRE(p.Cin > 0 && p.Cin <= MAX_NKB * BK, "xdw_conv: Cin must be at most 160 (the whole input window stays in shared memory)");
    SMK_REQUIRE(p.stride == 1 || (p.H % 2 == 0 && p.W % 2 == 0), "xdw_conv: stride 2 expects even input sizes (TF-SAME pad_begin 0)");
    SMK_REQUIRE(!p2 || (p2->B == p.B && p2->H == p.H && p2->W == p.W && p2->Cin == p.Cin && p2->mid == p.mid && p2->stride == p.stride &&
                        p2->round_out == p.round_out && !p2->w1t_lo == !p.w1t_lo && !p2->e_out == !p.e_out),
                "xdw_conv: paired problems must have identical shapes");
    const int Ho = (p.H + p.stride - 1) / p.stride, Wo = (p.W + p.stride - 1) / p.stride;
    const int TO = p.stride == 1 ? 14 : 7;
    XdwMaps mp;
    XdwArgs a{};
    for (int g = 0; g < nprob; ++g) {
        const XdwConv& q = g ? *p2 : p;
        if (int rc = encode_nhwc(&mp.x[g], q.x, q.B, q.H, q.W, q.Cin, q.Cin, WIN, 8, "xdw_conv(x)")) return rc;
        if (int rc = encode_2d(&mp.w[g], q.w1t, (uint64_t)q.mid, (uint64_t)q.Cin, (uint64_t)q.Cin, NC, "xdw_conv(w1)")) return rc;
        mp.wlo[g] = mp.w[g];
        if (q.w1t_lo) { if (int rc = encode_2d(&mp.wlo[g], q.w1t_lo, (uint64_t)q.mid, (uint64_t)q.Cin, (uint64_t)q.Cin, NC, "xdw_conv(w1 tails)")) return rc; }
        a.scale1[g] = q.scale1; a.bias1[g] = q.bias1; a.wdw[g] = q.wdw; a.scale2[g] = q.scale2; a.bias2[g] = q.bias2; a.out[g] = q.out;
        a.e_out[g] = q.e_out;
    }
    if (nprob == 1) {
        mp.x[1] = mp.x[0]; mp.w[1] = mp.w[0]; mp.wlo[1] = mp.wlo[0];
        a.scale1[1] = a.scale1[0]; a.bias1[1] = a.bias1[0]; a.wdw[1] = a.wdw[0]; a.scale2[1] = a.scale2[0]; a.bias2[1] = a.bias2[0]; a.out[1] = a.out[0];
        a.e_out[1] = a.e_out[0];
    }
    // Resident CTAs to aim for: one per SM (two fit for plain TF32 with Cin <= 64) leaves room on every SM for the other backbones' and batches'
    // kernels of the concurrent pipeline.
    const int slots = num_sms();
    a.H = p.H; a.W = p.W; a.Ho = Ho; a.Wo = Wo; a.mid = p.mid; a.nchunks = cdiv(p.mid, NC);
    {   // split the channel chunks over enough CTAs to fill the resident slots
        const long tiles = (long)nprob * cdiv(Wo, TO) * cdiv(Ho, TO) * p.B;
        int groups = (int)std::min<long>(a.nchunks, std::max<long>(1, (slots + tiles - 1) / tiles));
        a.chunks_per_group = cdiv(a.nchunks, groups);
        a.groups = cdiv(a.nchunks, a.chunks_per_group);
    }
    a.pad = p.stride == 1 ? 1 : 0;
    a.tiles_x = cdiv(Wo, TO); a.tiles_y = cdiv(Ho, TO);
    a.round_out = p.round_out;
    {
        const double px_in = (double)nprob * p.B * p.H * p.W, px_out = (double)nprob * p.B * Ho * Wo;
        const char* tag = p.w1t_lo ? "xdw_fused_tc3x" : "xdw_fused_tc";
        if (g_prof_detail) tag = prof_shape_tag(tag, (long)px_out, p.Cin, p.mid);
        SMK_TAG(tag, 4.0 * (px_in * p.Cin + px_out * p.mid + (double)nprob * p.mid * (p.Cin + 13)), 2.0 * px_in * p.Cin * p.mid + 18.0 * px_out * p.mid, st);
    }
    a.B = p.B;
    a.n_items = nprob * a.tiles_x * a.tiles_y * p.B * a.groups;
    {   // depthwise row grouping (dw_role): column runs x row groups over the slots of the schedule's depthwise threads
        const int ncols_e = Wo - (a.tiles_x - 1) * TO, nrows_e = Ho - (a.tiles_y - 1) * TO;
        const int dw_slots = (p.w1t_lo ? DW_THREADS : NUM_WORKERS) / (NC / 4), dwc = dw_cols(p.stride, p.w1t_lo != nullptr);
        auto group = [&](int ncols, int nrows) {
            const int n_rg = std::min(dw_slots / cdiv(ncols, dwc), nrows);
            return (unsigned)cdiv(nrows, n_rg) | (unsigned)n_rg << 4;
        };
        a.geom = group(TO, TO) | group(TO, nrows_e) << 8 | group(ncols_e, TO) << 16 | group(ncols_e, nrows_e) << 24;
    }
    const int grid = std::min(a.n_items, slots);         // persistent
    { int v = grid; a.d_grp = v % a.groups; v /= a.groups; a.d_tx = v % a.tiles_x; v /= a.tiles_x; a.d_ty = v % a.tiles_y; a.d_img = v / a.tiles_y; }
    if (p.w1t_lo) return p.stride == 1 ? launch_cin<1, 2>(p.Cin, mp, a, grid, st) : launch_cin<2, 2>(p.Cin, mp, a, grid, st);
    return p.stride == 1 ? launch_cin<1, 0>(p.Cin, mp, a, grid, st) : launch_cin<2, 0>(p.Cin, mp, a, grid, st);
}

}  // namespace smk

extern "C" int smk_debug_xdw(const float* x, int B, int H, int W, int Cin, const float* w1t, const float* scale1, const float* bias1,
                             int mid, const float* wdw, const float* scale2, const float* bias2, int stride, int round_out,
                             float* out, void* stream) {
    smk::XdwConv p{};
    p.x = x; p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.w1t = w1t; p.scale1 = scale1; p.bias1 = bias1; p.mid = mid; p.wdw = wdw;
    p.scale2 = scale2; p.bias2 = bias2; p.stride = stride; p.round_out = round_out; p.out = out;
    return smk::xdw_conv(p, (cudaStream_t)stream);
}

extern "C" int smk_debug_xdw3x(const float* x, int B, int H, int W, int Cin, const float* w1t_hi, const float* w1t_lo, const float* scale1,
                               const float* bias1, int mid, const float* wdw, const float* scale2, const float* bias2, int stride,
                               float* out, void* stream) {
    smk::XdwConv p{};
    p.x = x; p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.w1t = w1t_hi; p.w1t_lo = w1t_lo; p.scale1 = scale1; p.bias1 = bias1; p.mid = mid; p.wdw = wdw;
    p.scale2 = scale2; p.bias2 = bias2; p.stride = stride; p.round_out = 0; p.out = out;
    return smk::xdw_conv(p, (cudaStream_t)stream);
}
