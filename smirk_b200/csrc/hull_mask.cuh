// create_mask of the reference (datasets/base_dataset.py:9-15) for int32 points: OpenCV's convexHull (Sklansky's scan over
// the points sorted by x then y, clockwise = false, the output rotated so that the point indices ascend or descend where
// that is possible) followed by fillConvexPoly(mask, hull, 0) with lineType 8 and shift 0: every hull edge drawn as a
// clipped, left-to-right 8-connected Bresenham line, then one span per row from walking the two chains of edges out of
// the topmost vertex in 16.16 fixed point.  The clipping of an edge that leaves the image depends on which end is
// clipped first, so the hull's vertex order and start point are reproduced too.
// Written once for the host (tests compile it with a C++ compiler) and the device (video.cu's hull_mask_kernel).
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define SMK_HD __host__ __device__ __forceinline__
#else
#define SMK_HD inline
#endif

namespace smk {
namespace hull {

SMK_HD int sgn(long long v) { return (v > 0) - (v < 0); }

// Sklansky's scan from `start` towards `end` over the sorted points px[ord[k]], py[ord[k]]; returns the stack size.
SMK_HD int sklansky(const int* px, const int* py, const int* ord, int start, int end, int* stack, int nsign, int sign2) {
    const int incr = end > start ? 1 : -1;
    int pprev = start, pcur = pprev + incr, pnext = pcur + incr;
    int stacksize = 3;
    if (start == end || (px[ord[start]] == px[ord[end]] && py[ord[start]] == py[ord[end]])) {
        stack[0] = start;
        return 1;
    }
    stack[0] = pprev; stack[1] = pcur; stack[2] = pnext;
    end += incr;
    while (pnext != end) {
        const long long cury = py[ord[pcur]], nexty = py[ord[pnext]];
        const long long by = nexty - cury;
        if (sgn(by) != nsign) {
            const long long ax = (long long)px[ord[pcur]] - px[ord[pprev]];
            const long long bx = (long long)px[ord[pnext]] - px[ord[pcur]];
            const long long ay = cury - py[ord[pprev]];
            const long long convexity = ay * bx - ax * by;
            if (sgn(convexity) == sign2 && (ax != 0 || ay != 0)) {
                pprev = pcur; pcur = pnext; pnext += incr;
                stack[stacksize++] = pnext;
            } else if (pprev == start) {
                pcur = pnext; stack[1] = pcur; pnext += incr; stack[2] = pnext;
            } else {
                stack[stacksize - 2] = pnext;
                pcur = pprev; pprev = stack[stacksize - 4];
                stacksize--;
            }
        } else {
            pnext += incr;
            stack[stacksize - 1] = pnext;
        }
    }
    return --stacksize;
}

// convexHull(points, clockwise=false): ord = point indices sorted by (x, y); writes the hull's point indices to `out`,
// returns their count.  stack: n + 2 ints, tmp: n ints.
SMK_HD int convex_hull(const int* px, const int* py, const int* ord, int n, int* stack, int* out) {
    if (n <= 0) return 0;
    int miny_ind = 0, maxy_ind = 0, nout = 0;
    for (int i = 1; i < n; ++i) {
        const int y = py[ord[i]];
        if (py[ord[miny_ind]] > y) miny_ind = i;
        if (py[ord[maxy_ind]] < y) maxy_ind = i;
    }
    if (px[ord[0]] == px[ord[n - 1]] && py[ord[0]] == py[ord[n - 1]]) {
        out[nout++] = ord[0];
        return nout;
    }
    // upper half (counter-clockwise: the right chain first)
    int* tl_stack = stack;
    int tl_count = sklansky(px, py, ord, 0, maxy_ind, tl_stack, -1, 1);
    int* tr_stack = stack + tl_count;
    int tr_count = sklansky(px, py, ord, n - 1, maxy_ind, tr_stack, -1, -1);
    { int* t = tl_stack; tl_stack = tr_stack; tr_stack = t; int c = tl_count; tl_count = tr_count; tr_count = c; }
    for (int i = 0; i < tl_count - 1; ++i) out[nout++] = ord[tl_stack[i]];
    for (int i = tr_count - 1; i > 0; --i) out[nout++] = ord[tr_stack[i]];
    const int stop_idx = tr_count > 2 ? tr_stack[1] : tl_count > 2 ? tl_stack[tl_count - 2] : -1;
    // lower half
    int* bl_stack = stack;
    int bl_count = sklansky(px, py, ord, 0, miny_ind, bl_stack, 1, -1);
    int* br_stack = stack + bl_count;
    int br_count = sklansky(px, py, ord, n - 1, miny_ind, br_stack, 1, 1);
    if (stop_idx >= 0) {
        const int check_idx = bl_count > 2 ? bl_stack[1] : bl_count + br_count > 2 ? br_stack[2 - bl_count] : -1;
        if (check_idx == stop_idx || (check_idx >= 0 && px[ord[check_idx]] == px[ord[stop_idx]] &&
                                      py[ord[check_idx]] == py[ord[stop_idx]])) {
            // all points on one line: the lower chain is the upper one mirrored, except the extreme points
            bl_count = bl_count < 2 ? bl_count : 2;
            br_count = br_count < 2 ? br_count : 2;
        }
    }
    for (int i = 0; i < bl_count - 1; ++i) out[nout++] = ord[bl_stack[i]];
    for (int i = br_count - 1; i > 0; --i) out[nout++] = ord[br_stack[i]];
    // rotate so that the indices form an ascending or descending sequence where possible (the stack is free now)
    if (nout >= 3) {
        int min_idx = 0, max_idx = 0, lt = 0;
        for (int i = 1; i < nout; ++i) {
            const int idx = out[i];
            lt += out[i - 1] < idx;
            if (lt > 1 && lt <= i - 2) break;
            if (idx < out[min_idx]) min_idx = i;
            if (idx > out[max_idx]) max_idx = i;
        }
        const int mmdist = max_idx > min_idx ? max_idx - min_idx : min_idx - max_idx;
        if ((mmdist == 1 || mmdist == nout - 1) && (lt <= 1 || lt >= nout - 2)) {
            const int ascending = (max_idx + 1) % nout == min_idx;
            const int i0 = ascending ? min_idx : max_idx;
            int j = i0, i = 0;
            if (i0 > 0) {
                for (i = 0; i < nout; ++i) {
                    const int curr_idx = stack[i] = out[j];
                    const int next_j = j + 1 < nout ? j + 1 : 0;
                    const int next_idx = out[next_j];
                    if (i < nout - 1 && (ascending != (curr_idx < next_idx))) break;
                    j = next_j;
                }
                if (i == nout)
                    for (int k = 0; k < nout; ++k) out[k] = stack[k];
            }
        }
    }
    return nout;
}

// cv::clipLine for a w x h image (int64 arithmetic, the intersection truncated towards zero); false when outside.
SMK_HD bool clip_line(long long w, long long h, long long& x1, long long& y1, long long& x2, long long& y2) {
    const long long right = w - 1, bottom = h - 1;
    int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
    int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
        long long a;
        if (c1 & 12) {
            a = c1 < 8 ? 0 : bottom;
            x1 += (long long)((double)(a - y1) * (double)(x2 - x1) / (double)(y2 - y1));
            y1 = a;
            c1 = (x1 < 0) + (x1 > right) * 2;
        }
        if (c2 & 12) {
            a = c2 < 8 ? 0 : bottom;
            x2 += (long long)((double)(a - y2) * (double)(x2 - x1) / (double)(y2 - y1));
            y2 = a;
            c2 = (x2 < 0) + (x2 > right) * 2;
        }
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            if (c1) {
                a = c1 == 1 ? 0 : right;
                y1 += (long long)((double)(a - x1) * (double)(y2 - y1) / (double)(x2 - x1));
                x1 = a;
                c1 = 0;
            }
            if (c2) {
                a = c2 == 1 ? 0 : right;
                y2 += (long long)((double)(a - x2) * (double)(y2 - y1) / (double)(x2 - x1));
                x2 = a;
                c2 = 0;
            }
        }
    }
    return (c1 | c2) == 0;
}

// cv::line with connectivity 8 through a left-to-right LineIterator, clipped to the S x S image: set(x, y) per pixel.
template <class Set>
SMK_HD void line8(int S, int x1i, int y1i, int x2i, int y2i, Set set) {
    long long x1 = x1i, y1 = y1i, x2 = x2i, y2 = y2i;
    if ((unsigned)x1i >= (unsigned)S || (unsigned)x2i >= (unsigned)S || (unsigned)y1i >= (unsigned)S || (unsigned)y2i >= (unsigned)S)
        if (!clip_line(S, S, x1, y1, x2, y2)) return;
    int dx = (int)(x2 - x1), dy = (int)(y2 - y1), sx = 1, sy = 1;
    int px = (int)x1, py = (int)y1;
    if (dx < 0) { dx = -dx; dy = -dy; px = (int)x2; py = (int)y2; }
    if (dy < 0) { dy = -dy; sy = -1; }
    const bool vert = dy > dx;
    if (vert) { const int t = dx; dx = dy; dy = t; }
    int err = dx - (dy + dy);
    for (int k = 0; k <= dx; ++k) {
        set(px, py);
        const bool minor = err < 0;
        err += -(dy + dy) + (minor ? dx + dx : 0);
        if (vert) { py += sy; if (minor) px += sx; }
        else { px += sx; if (minor) py += sy; }
    }
}

// fillConvexPoly(img S x S, v[0..n), color, lineType 8, shift 0): line(x, y) per outline pixel, span(y, x0, x1) per row.
template <class Set, class Span>
SMK_HD void fill_convex_poly(int S, const int* vx, const int* vy, int n, Set set, Span span) {
    if (n <= 0) return;
    const long long ONE = 1LL << 16;
    int imin = 0;
    long long xmin = vx[0], xmax = vx[0], ymin = vy[0], ymax = vy[0];
    int p0x = vx[n - 1], p0y = vy[n - 1];
    for (int i = 0; i < n; ++i) {
        if (vy[i] < ymin) { ymin = vy[i]; imin = i; }
        ymax = ymax > vy[i] ? ymax : vy[i];
        xmax = xmax > vx[i] ? xmax : vx[i];
        xmin = xmin < vx[i] ? xmin : vx[i];
        line8(S, p0x, p0y, vx[i], vy[i], set);
        p0x = vx[i]; p0y = vy[i];
    }
    if (n < 3 || (int)xmax < 0 || (int)ymax < 0 || (int)xmin >= S || (int)ymin >= S) return;
    ymax = ymax < S - 1 ? ymax : S - 1;
    int e_idx[2] = {imin, imin}, e_di[2] = {1, n - 1}, e_ye[2];
    long long e_x[2] = {-ONE, -ONE}, e_dx[2] = {0, 0};
    int y = (int)ymin;
    e_ye[0] = e_ye[1] = y;
    int edges = n;
    do {
        for (int i = 0; i < 2; ++i) {
            if (y >= e_ye[i]) {
                int idx0 = e_idx[i];
                const int di = e_di[i];
                int idx = idx0 + di;
                if (idx >= n) idx -= n;
                for (; edges-- > 0;) {
                    const int ty = vy[idx];
                    if (ty > y) {
                        const long long xs = (long long)vx[idx0] << 16, xe = (long long)vx[idx] << 16;
                        e_ye[i] = ty;
                        e_dx[i] = ((xe - xs) * 2 + ((long long)ty - y)) / (2 * ((long long)ty - y));
                        e_x[i] = xs;
                        e_idx[i] = idx;
                        break;
                    }
                    idx0 = idx;
                    idx += di;
                    if (idx >= n) idx -= n;
                }
            }
        }
        if (edges < 0) break;
        if (y >= 0) {
            const int l = e_x[0] > e_x[1] ? 1 : 0, r = 1 - l;
            int xx1 = (int)((e_x[l] + (ONE >> 1)) >> 16), xx2 = (int)((e_x[r] + (ONE >> 1)) >> 16);
            if (xx2 >= 0 && xx1 < S) {
                if (xx1 < 0) xx1 = 0;
                if (xx2 >= S) xx2 = S - 1;
                span(y, xx1, xx2);
            }
        }
        e_x[0] += e_dx[0];
        e_x[1] += e_dx[1];
    } while (++y <= (int)ymax);
}

}  // namespace hull
}  // namespace smk
