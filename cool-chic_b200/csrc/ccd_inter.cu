// ccd_inter.cu -- P/B frame reconstruction on sm_90a (SURVEY 8 row a17 / f1).
//
// Replaces the P/B branch of decode_frame (bitstream/decode.py:156-189):
//   apply_global_translation  globalmotion.py:151-160   integer shift, border clamp
//   Warper.forward            warp.py:294-397           TRAINING branch (no 1/64-pel flow rounding),
//                                                       filter_size >= 6: windowed sinc (warp.py:226-268)
//                                                       filter_size 2 / 4: F.grid_sample bilinear / bicubic,
//                                                       border padding, align_corners (warp.py:50-56,314-334)
//   alpha / beta blending     decode.py:171-189
// One thread per pixel; the global shift is folded into the gather indices, so the shifted
// references are never materialised.  Same operation order as oracle/ccoracle.c::warp_sinc
// (coefficients in double -> fp32, fp32 products and sequential sums, no fusion).
#include <cuda_runtime.h>
#include <stdint.h>

#include "ccd_detmath.h"
#include "ccd_internal.h"

namespace {

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

template <int N>
__device__ __forceinline__ void sinc_coeffs(float s, float (&c)[N]) {
    const float PIf = 3.14159265358979323846f;
    constexpr int lt = -(N / 2) + 1;
#pragma unroll
    for (int k = 0; k < N; k++) {
        const float arg = __fsub_rn(s, (float)(lt + k));
        const float pa = __fmul_rn(PIf, arg);
        const double win = ccdm_cos((double)__fdiv_rn(pa, (float)N));
        const double sc = (arg == 0.0f) ? 1.0 : __ddiv_rn(ccdm_sin((double)pa), (double)pa);
        c[k] = __fmul_rn((float)win, (float)sc);
    }
}

// Reference planes: plane 0 is [h][w]; planes 1, 2 are [h >> cs][w >> cs] (cs = 1: a YUV 4:2:0 reference, read
// through the nearest x2 up-conversion of convert_420_to_444, io/format/yuv.py:303-316, folded into the gather
// index -- the 4:4:4 copy is never materialised).
struct RefPlanes {
    const float *p[3];
};
__device__ __forceinline__ float ref_at(const RefPlanes &r, int c, int cs, int w, int y, int x) {
    if (c == 0 || cs == 0) return __ldg(r.p[c] + (size_t)y * w + x);
    return __ldg(r.p[c] + (size_t)(y >> 1) * (w >> 1) + (x >> 1));
}

template <int N>
__device__ __forceinline__ void warp_pixel(const RefPlanes &ref, int cs, int h, int w, int gx, int gy, float fx,
                                           float fy, int x, int y, float (&out)[3]) {
    constexpr int lt = -(N / 2) + 1;
    const float rx = floorf(fx), ry = floorf(fy);
    float cx[N], cy[N];
    sinc_coeffs<N>(__fsub_rn(fx, rx), cx);
    sinc_coeffs<N>(__fsub_rn(fy, ry), cy);
    int xs[N], ys[N];
#pragma unroll
    for (int k = 0; k < N; k++) {
        float nx = __fadd_rn(__fadd_rn((float)x, (float)(lt + k)), rx);
        float ny = __fadd_rn(__fadd_rn((float)y, (float)(lt + k)), ry);
        nx = nx < 0.0f ? 0.0f : (nx > (float)(w - 1) ? (float)(w - 1) : nx);
        ny = ny < 0.0f ? 0.0f : (ny > (float)(h - 1) ? (float)(h - 1) : ny);
        xs[k] = clampi((int)nx + gx, 0, w - 1);
        ys[k] = clampi((int)ny + gy, 0, h - 1);
    }
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float col = 0.0f;
#pragma unroll
        for (int i = 0; i < N; i++) {
            float line = 0.0f;
#pragma unroll
            for (int j = 0; j < N; j++) {
                const float t = __fmul_rn(ref_at(ref, c, cs, w, ys[i], xs[j]), cx[j]);
                line = (j == 0) ? t : __fadd_rn(line, t);
            }
            const float t2 = __fmul_rn(line, cy[i]);
            col = (i == 0) ? t2 : __fadd_rn(col, t2);
        }
        out[c] = col;
    }
}

// torch.linspace(-1, 1, n)[i] as PyTorch's CPU kernel evaluates it (see oracle/ccoracle.c::lin_coord)
__device__ __forceinline__ float lin_coord(int n, int i) {
    const float step = __fdiv_rn(2.0f, (float)(n - 1));
    return (i < n / 2) ? __fmaf_rn(step, (float)i, -1.0f) : __fmaf_rn(-step, (float)(n - 1 - i), 1.0f);
}
__device__ __forceinline__ float cubic_near(float x) {
    const float a = __fsub_rn(__fmul_rn(1.25f, x), 2.25f);
    return __fmaf_rn(__fmul_rn(a, x), x, 1.0f);
}
__device__ __forceinline__ float cubic_far(float x) {
    const float a = __fadd_rn(__fmul_rn(-0.75f, x), 3.75f);
    const float b = __fadd_rn(__fmul_rn(a, x), -6.0f);
    return __fadd_rn(__fmul_rn(b, x), 3.0f);
}

// grid_sample(border, align_corners=True) of the globally shifted reference: N == 2 bilinear, N == 4 bicubic.
// Same operation order as oracle/ccoracle.c::warp_grid.
template <int N>
__device__ __forceinline__ void grid_pixel(const RefPlanes &ref, int cs, int h, int w, int gx, int gy, float fx,
                                           float fy, int x, int y, float (&out)[3]) {
    const float sx = (float)((w - 1.0) / 2.0), sy = (float)((h - 1.0) / 2.0);
    const float g0 = __fadd_rn(lin_coord(w, x), __fdiv_rn(fx, sx)), g1 = __fadd_rn(lin_coord(h, y), __fdiv_rn(fy, sy));
    float ix = __fmul_rn(__fadd_rn(g0, 1.0f), sx), iy = __fmul_rn(__fadd_rn(g1, 1.0f), sy);
    if (N == 2) {
        ix = fminf((float)(w - 1), fmaxf(ix, 0.0f));
        iy = fminf((float)(h - 1), fmaxf(iy, 0.0f));
        const float xw = floorf(ix), yn = floorf(iy);
        const float ww = __fsub_rn(ix, xw), e = __fsub_rn(1.0f, ww), nn = __fsub_rn(iy, yn), s = __fsub_rn(1.0f, nn);
        const float k_nw = __fmul_rn(s, e), k_ne = __fmul_rn(s, ww), k_sw = __fmul_rn(nn, e), k_se = __fmul_rn(nn, ww);
        const int x0 = (int)xw, y0 = (int)yn, x1 = x0 + 1, y1 = y0 + 1;
        const int xa = clampi(x0 + gx, 0, w - 1), xb = clampi((x1 < w ? x1 : w - 1) + gx, 0, w - 1);
        const int ya = clampi(y0 + gy, 0, h - 1), yb = clampi((y1 < h ? y1 : h - 1) + gy, 0, h - 1);
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float v00 = ref_at(ref, c, cs, w, ya, xa);
            const float v01 = x1 < w ? ref_at(ref, c, cs, w, ya, xb) : 0.0f;
            const float v10 = y1 < h ? ref_at(ref, c, cs, w, yb, xa) : 0.0f;
            const float v11 = (x1 < w && y1 < h) ? ref_at(ref, c, cs, w, yb, xb) : 0.0f;
            float r = __fmul_rn(v00, k_nw);
            r = __fmaf_rn(v01, k_ne, r);
            r = __fmaf_rn(v10, k_sw, r);
            r = __fmaf_rn(v11, k_se, r);
            out[c] = r;
        }
    } else {
        const float fxx = floorf(ix), fyy = floorf(iy);
        const float tx = __fsub_rn(ix, fxx), ty = __fsub_rn(iy, fyy);
        const float cx[4] = {cubic_far(__fadd_rn(tx, 1.0f)), cubic_near(tx), cubic_near(__fsub_rn(1.0f, tx)),
                             cubic_far(__fsub_rn(2.0f, tx))};
        const float cy[4] = {cubic_far(__fadd_rn(ty, 1.0f)), cubic_near(ty), cubic_near(__fsub_rn(1.0f, ty)),
                             cubic_far(__fsub_rn(2.0f, ty))};
        int xs[4], ys[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const float nx = fminf((float)(w - 1), fmaxf(__fadd_rn(fxx, (float)(k - 1)), 0.0f));
            const float ny = fminf((float)(h - 1), fmaxf(__fadd_rn(fyy, (float)(k - 1)), 0.0f));
            xs[k] = clampi((int)nx + gx, 0, w - 1);
            ys[k] = clampi((int)ny + gy, 0, h - 1);
        }
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float rows[4];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                float r = __fmul_rn(cx[0], ref_at(ref, c, cs, w, ys[i], xs[0]));
                r = __fmaf_rn(cx[1], ref_at(ref, c, cs, w, ys[i], xs[1]), r);
                r = __fmaf_rn(cx[2], ref_at(ref, c, cs, w, ys[i], xs[2]), r);
                r = __fmaf_rn(cx[3], ref_at(ref, c, cs, w, ys[i], xs[3]), r);
                rows[i] = r;
            }
            float a = __fmul_rn(cy[0], rows[0]);
            a = __fmaf_rn(cy[1], rows[1], a);
            a = __fmaf_rn(cy[2], rows[2], a);
            a = __fmaf_rn(cy[3], rows[3], a);
            out[c] = a;
        }
    }
}

template <int N>
__device__ __forceinline__ void predict_pixel(const RefPlanes &ref, int cs, int h, int w, int gx, int gy, float fx,
                                              float fy, int x, int y, float (&out)[3]) {
    if constexpr (N <= 4)
        grid_pixel<N>(ref, cs, h, w, gx, gy, fx, fy, x, y, out);
    else
        warp_pixel<N>(ref, cs, h, w, gx, gy, fx, fy, x, y, out);
}

// One thread per pixel; a warp covers a 16 x 2 patch (lane = lx + 16 ly), so that the 2 x 2 chroma blocks of a
// 4:2:0 frame sit inside one warp and the frame tail of decode_frame (bitstream/decode.py:191-206: round ->
// 2 x 2 average of U, V -> clamp -> round) is done with four shuffles instead of a second pass over HBM.
//   M == 0: out[c] = pre-rounding frame (three full planes)
//   M  > 0: out[c] = finished frame on the k / M grid; out_420: U, V planes are [h/2][w/2]
template <int N>
__global__ void __launch_bounds__(128)
    k_inter_predict(const float *__restrict__ residue, const float *__restrict__ motion, RefPlanes ref0, RefPlanes ref1,
                    int ref_cs, int h, int w, int is_b, int g0x, int g0y, int g1x, int g1y, float M, int out_420,
                    float *__restrict__ o0, float *__restrict__ o1, float *__restrict__ o2) {
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int px = blockIdx.x * 32 + (wrp & 1) * 16 + (lane & 15);
    const int py = blockIdx.y * 4 + (wrp >> 1) * 2 + (lane >> 4);
    const bool inside = px < w && py < h;
    const int x = px < w ? px : w - 1, y = py < h ? py : h - 1;  // every lane computes (shuffles below)
    const size_t plane = (size_t)h * w, i = (size_t)y * w + x;
    float p0[3], p1[3] = {0.0f, 0.0f, 0.0f};
    predict_pixel<N>(ref0, ref_cs, h, w, g0x, g0y, motion[i], motion[plane + i], x, y, p0);
    float beta = 0.0f;
    if (is_b) {
        predict_pixel<N>(ref1, ref_cs, h, w, g1x, g1y, motion[2 * plane + i], motion[3 * plane + i], x, y, p1);
        beta = __fadd_rn(residue[4 * plane + i], 0.5f);
        beta = clamp01(beta);
    }
    float alpha = clamp01(__fadd_rn(residue[3 * plane + i], 0.5f));
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float pred = p0[c];
        if (is_b) pred = __fadd_rn(__fmul_rn(beta, pred), __fmul_rn(__fsub_rn(1.0f, beta), p1[c]));
        v[c] = __fadd_rn(__fmul_rn(alpha, pred), residue[c * plane + i]);
    }
    float *const outp[3] = {o0, o1, o2};
    if (M == 0.0f) {
        if (inside) {
#pragma unroll
            for (int c = 0; c < 3; c++) outp[c][i] = v[c];
        }
        return;
    }
#pragma unroll
    for (int c = 0; c < 3; c++) v[c] = quant(v[c], M);
    if (!out_420) {
        if (inside) {
#pragma unroll
            for (int c = 0; c < 3; c++) outp[c][i] = quant(clamp01(v[c]), M);
        }
        return;
    }
    if (inside) o0[i] = quant(clamp01(v[0]), M);
    // 2 x 2 average of the rounded chroma samples, in the order of F.avg_pool2d's reference loop (yuv.py:295)
    const int base = lane & ~17;
#pragma unroll
    for (int c = 1; c < 3; c++) {
        float s = 0.0f;
        s = __fadd_rn(s, __shfl_sync(0xffffffffu, v[c], base));
        s = __fadd_rn(s, __shfl_sync(0xffffffffu, v[c], base + 1));
        s = __fadd_rn(s, __shfl_sync(0xffffffffu, v[c], base + 16));
        s = __fadd_rn(s, __shfl_sync(0xffffffffu, v[c], base + 17));
        if (lane == base && px + 1 < w && py + 1 < h)
            outp[c][(size_t)(py >> 1) * (w >> 1) + (px >> 1)] = quant(clamp01(__fdiv_rn(s, 4.0f)), M);
    }
}

// Statistics of the P/B prediction (training/test.py:169-199), one thread per pixel of a 32 x 4 tile: p0, p1, beta,
// alpha and pred with exactly the fp32 operations of k_inter_predict, and with a source orig = ks / M (4:2:0 chroma
// read at >> 1, convert_420_to_444) and dummy = ((0 + r0) + r1) / n_refs.  Per-pixel f64 terms, then a fixed-order
// tree over the CTA: one partial per CTA and per sum, added by the host in tile order (the same value on every run).
template <int N>
__global__ void __launch_bounds__(128)
    k_inter_stats(const float *__restrict__ residue, const float *__restrict__ motion, RefPlanes ref0, RefPlanes ref1,
                  int ref_cs, int h, int w, int is_b, int g0x, int g0y, int g1x, int g1y, InterStatsOut o) {
    __shared__ double red[4][128];
    const int t = threadIdx.x;
    const int x = blockIdx.x * 32 + (t & 31), y = blockIdx.y * 4 + (t >> 5);
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    if (x < w && y < h) {
        const size_t plane = (size_t)h * w, i = (size_t)y * w + x;
        float p0[3], p1[3] = {0.0f, 0.0f, 0.0f};
        predict_pixel<N>(ref0, ref_cs, h, w, g0x, g0y, motion[i], motion[plane + i], x, y, p0);
        float beta = 0.0f;
        if (is_b) {
            predict_pixel<N>(ref1, ref_cs, h, w, g1x, g1y, motion[2 * plane + i], motion[3 * plane + i], x, y, p1);
            beta = __fadd_rn(residue[4 * plane + i], 0.5f);
            beta = clamp01(beta);
        }
        const float alpha = clamp01(__fadd_rn(residue[3 * plane + i], 0.5f));
        float pred[3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
            pred[c] = p0[c];
            if (is_b) pred[c] = __fadd_rn(__fmul_rn(beta, pred[c]), __fmul_rn(__fsub_rn(1.0f, beta), p1[c]));
        }
        acc[0] = alpha;
        acc[1] = beta;
        if (o.src) {
            const size_t wc = (size_t)(w >> ref_cs), nc = (size_t)(h >> ref_cs) * wc;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const size_t k = o.src_hwc ? 3 * i + c
                                           : (c == 0 ? i : plane + (c - 1) * nc + (size_t)(y >> ref_cs) * wc + (x >> ref_cs));
                const int ks = o.src_wide ? (int)__ldg(static_cast<const uint16_t *>(o.src) + k)
                                          : (int)__ldg(static_cast<const uint8_t *>(o.src) + k);
                const float orig = __fdiv_rn((float)ks, o.src_M);
                float dummy = __fadd_rn(0.0f, ref_at(ref0, c, ref_cs, w, y, x));
                if (is_b) dummy = __fadd_rn(dummy, ref_at(ref1, c, ref_cs, w, y, x));
                dummy = __fdiv_rn(dummy, is_b ? 2.0f : 1.0f);
                const float e = __fsub_rn(pred[c], orig), f = __fsub_rn(dummy, orig);
                acc[2] += (double)__fmul_rn(e, e);
                acc[3] += (double)__fmul_rn(f, f);
            }
        }
        if (o.alpha) o.alpha[i] = alpha;
        if (o.beta) o.beta[i] = beta;
        if (o.pred) {
#pragma unroll
            for (int c = 0; c < 3; c++) o.pred[c * plane + i] = pred[c];
        }
    }
#pragma unroll
    for (int k = 0; k < 4; k++) red[k][t] = acc[k];
    __syncthreads();
    for (int s = 64; s > 0; s >>= 1) {
        if (t < s) {
#pragma unroll
            for (int k = 0; k < 4; k++) red[k][t] += red[k][t + s];
        }
        __syncthreads();
    }
    if (t < 4) o.part[4 * ((size_t)blockIdx.y * gridDim.x + blockIdx.x) + t] = red[t][0];
}

}  // namespace

int64_t ccd_inter_stats_ctas(int h, int w) { return (int64_t)((w + 31) / 32) * ((h + 3) / 4); }

int ccd_inter_stats_launch(const InterLaunch &a, const InterStatsOut &o, cudaStream_t st) {
    const dim3 block(128, 1, 1), grid((a.w + 31) / 32, (a.h + 3) / 4, 1);
    RefPlanes r0, r1;
    for (int c = 0; c < 3; c++) {
        r0.p[c] = a.ref0[c];
        r1.p[c] = a.ref1[c] ? a.ref1[c] : a.ref0[c];
    }
#define LAUNCH(N)                                                                                                  \
    k_inter_stats<N><<<grid, block, 0, st>>>(a.residue, a.motion, r0, r1, a.ref_cs, a.h, a.w, a.is_b, a.gf[0], a.gf[1], \
                                             a.gf[2], a.gf[3], o)
    switch (a.filter_size) {
        case 2: if (a.h < 2 || a.w < 2) return -1; LAUNCH(2); break;
        case 4: if (a.h < 2 || a.w < 2) return -1; LAUNCH(4); break;
        case 6: LAUNCH(6); break;
        case 8: LAUNCH(8); break;
        case 10: LAUNCH(10); break;
        case 12: LAUNCH(12); break;
        case 14: LAUNCH(14); break;
        default: return -1;
    }
#undef LAUNCH
    g_ccd_launches++;
    return (int)cudaGetLastError();
}

int ccd_inter_launch(const InterLaunch &a, cudaStream_t st) {
    const dim3 block(128, 1, 1), grid((a.w + 31) / 32, (a.h + 3) / 4, 1);
    RefPlanes r0, r1;
    for (int c = 0; c < 3; c++) {
        r0.p[c] = a.ref0[c];
        r1.p[c] = a.ref1[c] ? a.ref1[c] : a.ref0[c];
    }
#define LAUNCH(N)                                                                                                  \
    k_inter_predict<N><<<grid, block, 0, st>>>(a.residue, a.motion, r0, r1, a.ref_cs, a.h, a.w, a.is_b, a.gf[0],    \
                                               a.gf[1], a.gf[2], a.gf[3], a.M, a.out_420, a.out[0], a.out[1], a.out[2])
    switch (a.filter_size) {
        case 2: if (a.h < 2 || a.w < 2) return -1; LAUNCH(2); break;
        case 4: if (a.h < 2 || a.w < 2) return -1; LAUNCH(4); break;
        case 6: LAUNCH(6); break;
        case 8: LAUNCH(8); break;
        case 10: LAUNCH(10); break;
        case 12: LAUNCH(12); break;
        case 14: LAUNCH(14); break;  // the largest size the 4-bit header field can carry (header.py:217)
        default: return -1;
    }
#undef LAUNCH
    g_ccd_launches++;
    return (int)cudaGetLastError();
}
