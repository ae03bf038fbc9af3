// latlong.cu -- equirectangular (latitude-longitude) panoramas to cube maps and the adjoint (DESIGN.md §7.13).
//
// Forward: one thread per cube texel (item, face, row, column): the fp32 mean of the n x n bilinear lookups of the
// panorama at the texel's sub-sample directions, summed in registers in row-major order.  For C = 1 .. 4 the panorama
// texels arrive as one vector load (C = 2, 4, aligned) and the cube texel leaves as a vector store, or for C = 3 through
// the warp's slice of shared memory (stage_store); any other C goes one channel at a time.
// Backward: a gather, one thread per panorama texel and item.  The samples whose taps can touch the texel lie, on each
// face, in a box of face coordinates taken from the texel's footprint in (theta, phi), widened by a slack; every sample
// in the box has its taps recomputed exactly as the forward computes them, so the adjoint sums exactly the forward's
// (sample, texel) pairs, in a fixed order (face, sample row, sample column, tap) and with no atomics.
#include "../../include/dirt_b200.h"
#include "common.cuh"

#include <cmath>
#include <type_traits>

namespace dirt {

namespace {

constexpr int LL_THREADS = 256;
// grid caps (grid-stride loops beyond them); a build may lower them to test those loops
#ifndef DIRT_LATLONG_MAX_BLOCKS
#define DIRT_LATLONG_MAX_BLOCKS 65536
#endif
#ifndef DIRT_LATLONG_MAX_ITEMS
#define DIRT_LATLONG_MAX_ITEMS 65535
#endif
constexpr long long LL_MAX_BLOCKS = DIRT_LATLONG_MAX_BLOCKS;
constexpr int LL_MAX_ITEMS = DIRT_LATLONG_MAX_ITEMS;   // gridDim.y of the adjoint
constexpr float LL_INV_2PI = (float)(0.5 / M_PI);      // 0.15915494f, rounded once
constexpr float LL_INV_PI = (float)(1.0 / M_PI);       // 0.31830987f
constexpr double LL_PI = M_PI;

// The panorama taps of one sample: padded row r0 = floor(pr) read as panorama rows ra = clamp(r0 - 1) and
// rb = clamp(r0) (the padding repeats rows 0 and H-1), columns c0, c1 modulo W, and the fractions.
struct LlTaps {
    int ra, rb, c0, c1;
    float fr, fc;
};

// Sample (i, j) of face f, i along tc and j along sc, i, j in 0 .. S*n - 1 and den = S*n: each operation rounded in
// fp32 in the order of tests/latlong_restatement.py.
__device__ __forceinline__ LlTaps latlong_taps(int f, int i, int j, float den, int H, int W)
{
    const float sc = __fsub_rn(__fdiv_rn((float)(2 * j + 1), den), 1.0f);
    const float tc = __fsub_rn(__fdiv_rn((float)(2 * i + 1), den), 1.0f);
    float x, y, z;
    face_point(f, sc, tc, x, y, z);
    const float phi = atan2f(x, -z);
    const float theta = atan2f(__fsqrt_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z))), y);
    const float u = __fadd_rn(__fmul_rn(phi, LL_INV_2PI), 0.5f);
    const float v = __fmul_rn(theta, LL_INV_PI);
    const float pc = __fsub_rn(__fmul_rn(u, (float)W), 0.5f);
    const float pr = __fadd_rn(__fsub_rn(__fmul_rn(v, (float)H), 0.5f), 1.0f);
    const float flr = floorf(pr), flc = floorf(pc);
    LlTaps t;
    t.fr = __fsub_rn(pr, flr);
    t.fc = __fsub_rn(pc, flc);
    const int r0 = (int)flr;   // 0 .. H: theta is in [0, pi] up to rounding
    t.ra = min(max(r0 - 1, 0), H - 1);
    t.rb = min(max(r0, 0), H - 1);
    int c0 = (int)flc % W;
    c0 = c0 < 0 ? c0 + W : c0;
    t.c0 = c0;
    t.c1 = c0 + 1 == W ? 0 : c0 + 1;
    return t;
}

struct LlDims {
    int TB, H, W, S, C, n;
};

// One thread per cube texel, CT = C in 1 .. 4, or 0 for any C (one channel at a time, scalar accesses).  VEC: the
// panorama and the cube map are aligned for the vector loads and stores.  The loop runs per warp, so that the C = 3
// staging sees all 32 lanes.
template <int CT, bool VEC>
__global__ void __launch_bounds__(LL_THREADS) latlong_forward_kernel(const float* __restrict__ panorama,
                                                                     float* __restrict__ cubemap, LlDims d)
{
    constexpr int NV = CT ? CT : 1;
    const int C = CT ? CT : d.C;
    __shared__ __align__(16) float stage[CT == 3 ? LL_THREADS * 3 : 1];
    const int lane = threadIdx.x & 31;
    const int S = d.S, n = d.n;
    const long long face_texels = (long long)S * S, total = (long long)d.TB * 6 * face_texels;
    const long long stride = (long long)gridDim.x * LL_THREADS;
    const float den = (float)(S * n), nn = (float)(n * n);
    for (long long base = (long long)blockIdx.x * LL_THREADS + (threadIdx.x & ~31); base < total; base += stride) {
        const long long e = base + lane;
        const bool valid = e < total;
        const long long tf = valid ? e / face_texels : 0;   // item * 6 + face
        const int rc = valid ? (int)(e - tf * face_texels) : 0, r = rc / S, c = rc - r * S, f = (int)(tf % 6);
        const float* pan = panorama + (tf / 6) * d.H * (long long)d.W * C;
        for (int c0 = 0; c0 < C; c0 += NV) {
            float acc[NV];
#pragma unroll
            for (int k = 0; k < NV; ++k) acc[k] = 0.f;
            if (valid) {
                for (int a = 0; a < n; ++a) {
                    for (int b = 0; b < n; ++b) {
                        const LlTaps t = latlong_taps(f, r * n + a, c * n + b, den, d.H, d.W);
                        float t00[NV], t01[NV], t10[NV], t11[NV];
                        load_row<NV, VEC>(pan + ((long long)t.ra * d.W + t.c0) * C + c0, t00);
                        load_row<NV, VEC>(pan + ((long long)t.ra * d.W + t.c1) * C + c0, t01);
                        load_row<NV, VEC>(pan + ((long long)t.rb * d.W + t.c0) * C + c0, t10);
                        load_row<NV, VEC>(pan + ((long long)t.rb * d.W + t.c1) * C + c0, t11);
#pragma unroll
                        for (int k = 0; k < NV; ++k)
                            acc[k] = __fadd_rn(acc[k], bilinear(t00[k], t01[k], t10[k], t11[k], t.fr, t.fc));
                    }
                }
            }
            float v[NV];
#pragma unroll
            for (int k = 0; k < NV; ++k) v[k] = __fdiv_rn(acc[k], nn);
            float* o = cubemap + e * C + c0;
            if (VEC && CT == 4) {
                if (valid) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1 % NV], v[2 % NV], v[3 % NV]);
            } else if (VEC && CT == 2) {
                if (valid) *reinterpret_cast<float2*>(o) = make_float2(v[0], v[1 % NV]);
            } else if (CT == 3) {
                const int m = total - base < 32 ? (int)(total - base) : 32;
                stage_store<NV>(cubemap, base, m, stage + (threadIdx.x & ~31) * 3, lane, v);
            } else if (valid) {
#pragma unroll
                for (int k = 0; k < NV; ++k) o[k] = v[k];
            }
        }
    }
}

// ---- the adjoint's candidate boxes ----------------------------------------------------------------------------------
//
// A panorama texel (R, Q) is read by the samples whose padded row r0 is R or R + 1 and whose column c0 is Q - 1 or Q
// (mod W): v H in [R - 1/2, R + 3/2) and u W in [Q - 1/2, Q + 3/2) (mod W).  With a margin for the forward's fp32
// rounding that is the cell theta in [th0, th1], phi in [ph0, ph1] below.  On the side faces (+-X, +-Z) the face
// coordinates are sc = -tan(phi - phi_f) and tc = -cot(theta) sqrt(1 + sc^2); on +-Y, sc and tc are rho sin(phi) and
// -+rho cos(phi) (+Y) or rho cos(phi) (-Y) with rho = tan of the angle from the pole.  Each bound below is taken over
// the product of the ranges, so it holds every point of the cell; float64.

// sin over [a0, a1]
__device__ __forceinline__ void sin_range(double a0, double a1, double& lo, double& hi)
{
    if (a1 - a0 >= 2.0 * LL_PI) {
        lo = -1.0;
        hi = 1.0;
        return;
    }
    const double s0 = sin(a0), s1 = sin(a1);
    lo = fmin(s0, s1);
    hi = fmax(s0, s1);
    // the interval holds pi/2 + 2 pi k, or -pi/2 + 2 pi k
    if (0.5 * LL_PI + 2.0 * LL_PI * ceil((a0 - 0.5 * LL_PI) / (2.0 * LL_PI)) <= a1) hi = 1.0;
    if (-0.5 * LL_PI + 2.0 * LL_PI * ceil((a0 + 0.5 * LL_PI) / (2.0 * LL_PI)) <= a1) lo = -1.0;
}

struct LlBox {
    int i0, i1, j0, j1;   // sample rows i0 .. i1 and columns j0 .. j1 (empty when i0 > i1 or j0 > j1)
};

// [lo, hi] of a face coordinate -> the sample indices k whose (2k + 1) / Sn - 1 can fall there
__device__ __forceinline__ void index_range(double lo, double hi, int Sn, int& k0, int& k1)
{
    // 2.5e-7 covers the fp32 rounding of a sample's coordinate, 1e-3 of an index float64's of the bounds
    lo = fmin(fmax(lo - 2.5e-7, -2.0), 2.0);
    hi = fmax(fmin(hi + 2.5e-7, 2.0), -2.0);
    k0 = max((int)ceil(((lo + 1.0) * Sn - 1.0) * 0.5 - 1e-3), 0);
    k1 = min((int)floor(((hi + 1.0) * Sn - 1.0) * 0.5 + 1e-3), Sn - 1);
}

__device__ __forceinline__ LlBox face_box(int f, double th0, double th1, double ph0, double ph1, int Sn)
{
    LlBox b = {1, 0, 1, 0};
    double s_lo, s_hi, t_lo, t_hi;
    if (f == 2 || f == 3) {
        // angle from the pole, within atan(sqrt(2)) on the face
        const double pole_max = 0.9553166181245093 + 1e-3;
        const double a0 = f == 2 ? fmax(th0, 0.0) : fmax(LL_PI - th1, 0.0);
        const double a1 = fmin(f == 2 ? th1 : LL_PI - th0, pole_max);
        if (a0 > a1) return b;
        const double r0 = tan(a0), r1 = tan(a1);
        double sn0, sn1, cs0, cs1;
        sin_range(ph0, ph1, sn0, sn1);
        sin_range(ph0 + 0.5 * LL_PI, ph1 + 0.5 * LL_PI, cs0, cs1);   // cos
        s_lo = fmin(r0 * sn0, r1 * sn0);
        s_hi = fmax(r0 * sn1, r1 * sn1);
        const double c_lo = fmin(r0 * cs0, r1 * cs0), c_hi = fmax(r0 * cs1, r1 * cs1);
        t_lo = f == 2 ? -c_hi : c_lo;
        t_hi = f == 2 ? -c_lo : c_hi;
    } else {
        const double phi_f = f == 0 ? 0.5 * LL_PI : f == 1 ? -0.5 * LL_PI : f == 4 ? LL_PI : 0.0;
        const double edge = 0.25 * LL_PI + 1e-3;
        double d0 = -edge, d1 = edge;
        if (ph1 - ph0 < 0.5 * LL_PI) {
            // the one copy of the interval (mod 2 pi) that can meet the face's quarter
            const double k = rint((0.5 * (ph0 + ph1) - phi_f) / (2.0 * LL_PI));
            d0 = fmax(ph0 - phi_f - 2.0 * LL_PI * k, -edge);
            d1 = fmin(ph1 - phi_f - 2.0 * LL_PI * k, edge);
            if (d0 > d1) return b;
        }
        s_lo = -tan(d1);
        s_hi = -tan(d0);
        const double q0 = s_lo <= 0.0 && s_hi >= 0.0 ? 1.0 : sqrt(1.0 + fmin(s_lo * s_lo, s_hi * s_hi));
        const double q1 = sqrt(1.0 + fmax(s_lo * s_lo, s_hi * s_hi));
        // -cot(theta), increasing on (0, pi)
        const double m0 = th0 <= 0.0 ? -INFINITY : -cos(th0) / sin(th0);
        const double m1 = th1 >= LL_PI ? INFINITY : -cos(th1) / sin(th1);
        t_lo = fmin(m0 * q0, m0 * q1);
        t_hi = fmax(m1 * q0, m1 * q1);
    }
    index_range(s_lo, s_hi, Sn, b.j0, b.j1);
    index_range(t_lo, t_hi, Sn, b.i0, b.i1);
    return b;
}

// One thread per panorama texel (grid-stride) and item (gridDim.y, item-stride), channels c0 .. c0 + NV - 1:
// grad_panorama = sum over the forward's (sample, tap) pairs on this texel of the tap's weight times
// grad_cubemap / n^2, in the order face, sample row, sample column, tap (00, 01, 10, 11).
template <int NV>
__global__ void __launch_bounds__(LL_THREADS) latlong_backward_kernel(const float* __restrict__ grad_cubemap,
                                                                      float* __restrict__ grad_panorama, LlDims d, int c0)
{
    const int S = d.S, n = d.n, Sn = S * n, H = d.H, W = d.W, C = d.C;
    const long long texels = (long long)H * W, stride = (long long)gridDim.x * LL_THREADS;
    const float den = (float)Sn, nn = (float)(n * n);
    // margins in rows and columns for the forward's fp32 coordinates (good to a few 1e-7 relative)
    const double mr = 0.05 + 4e-6 * H, mc = 0.05 + 4e-6 * W;
    for (long long e = (long long)blockIdx.x * LL_THREADS + threadIdx.x; e < texels; e += stride) {
        const int R = (int)(e / W), Q = (int)(e - (long long)R * W);
        const double th0 = (R - 0.5 - mr) * LL_PI / H, th1 = (R + 1.5 + mr) * LL_PI / H;
        const double ph0 = (Q - 0.5 - mc) * 2.0 * LL_PI / W - LL_PI, ph1 = (Q + 1.5 + mc) * 2.0 * LL_PI / W - LL_PI;
        for (int tb = blockIdx.y; tb < d.TB; tb += gridDim.y) {
            const float* g = grad_cubemap + (long long)tb * 6 * S * S * C + c0;
            float acc[NV];
#pragma unroll
            for (int k = 0; k < NV; ++k) acc[k] = 0.f;
            for (int f = 0; f < 6; ++f) {
                const LlBox b = face_box(f, th0, th1, ph0, ph1, Sn);
                for (int i = b.i0; i <= b.i1; ++i) {
                    for (int j = b.j0; j <= b.j1; ++j) {
                        const LlTaps t = latlong_taps(f, i, j, den, H, W);
                        const bool ra = t.ra == R, rb = t.rb == R, q0 = t.c0 == Q, q1 = t.c1 == Q;
                        if (!((ra || rb) && (q0 || q1))) continue;
                        const float omr = __fsub_rn(1.0f, t.fr), omc = __fsub_rn(1.0f, t.fc);
                        const long long texel = ((long long)f * S + i / n) * S + j / n;
                        float gs[NV];
#pragma unroll
                        for (int k = 0; k < NV; ++k) gs[k] = __fdiv_rn(__ldg(g + texel * C + k), nn);
                        auto add = [&](float w) {
#pragma unroll
                            for (int k = 0; k < NV; ++k) acc[k] = __fadd_rn(acc[k], __fmul_rn(gs[k], w));
                        };
                        if (ra && q0) add(__fmul_rn(omc, omr));
                        if (ra && q1) add(__fmul_rn(t.fc, omr));
                        if (rb && q0) add(__fmul_rn(omc, t.fr));
                        if (rb && q1) add(__fmul_rn(t.fc, t.fr));
                    }
                }
            }
            float* o = grad_panorama + ((long long)tb * texels + e) * C + c0;
#pragma unroll
            for (int k = 0; k < NV; ++k) o[k] = acc[k];
        }
    }
}

inline unsigned ll_blocks(long long work)
{
    const long long b = (work + LL_THREADS - 1) / LL_THREADS;
    return (unsigned)(b < LL_MAX_BLOCKS ? (b > 0 ? b : 1) : LL_MAX_BLOCKS);
}

inline bool aligned_to(const void* p, int bytes) { return (uintptr_t)p % bytes == 0; }

template <int CT>
cudaError_t latlong_forward_ct(const float* panorama, float* cubemap, const LlDims& d, cudaStream_t stream)
{
    const unsigned blocks = ll_blocks((long long)d.TB * 6 * d.S * d.S);
    constexpr int bytes = CT == 4 ? 16 : CT == 2 ? 8 : 4;
    if (CT == 2 || CT == 4) {
        if (aligned_to(panorama, bytes) && aligned_to(cubemap, bytes))
            latlong_forward_kernel<CT, true><<<blocks, LL_THREADS, 0, stream>>>(panorama, cubemap, d);
        else
            latlong_forward_kernel<CT, false><<<blocks, LL_THREADS, 0, stream>>>(panorama, cubemap, d);
    } else {
        latlong_forward_kernel<CT, false><<<blocks, LL_THREADS, 0, stream>>>(panorama, cubemap, d);
    }
    return launched();
}

}  // namespace

int latlong_samples(int H, int W, int S)
{
    const double m = W > 2 * (double)H ? (double)W : 2.0 * H;
    const double n = ceil(m / (M_PI * S));
    return n > 1.0 ? (int)n : 1;
}

cudaError_t launch_latlong_forward(const float* panorama, float* cubemap, int TB, int H, int W, int S, int C,
                                   cudaStream_t stream)
{
    const LlDims d = {TB, H, W, S, C, latlong_samples(H, W, S)};
    switch (C) {
        case 1: return latlong_forward_ct<1>(panorama, cubemap, d, stream);
        case 2: return latlong_forward_ct<2>(panorama, cubemap, d, stream);
        case 3: return latlong_forward_ct<3>(panorama, cubemap, d, stream);
        case 4: return latlong_forward_ct<4>(panorama, cubemap, d, stream);
        default: return latlong_forward_ct<0>(panorama, cubemap, d, stream);
    }
}

cudaError_t launch_latlong_backward(const float* grad_cubemap, float* grad_panorama, int TB, int H, int W, int S, int C,
                                    cudaStream_t stream)
{
    const LlDims d = {TB, H, W, S, C, latlong_samples(H, W, S)};
    const dim3 grid(ll_blocks((long long)H * W), TB < LL_MAX_ITEMS ? TB : LL_MAX_ITEMS);
    for (int c0 = 0; c0 < C; c0 += 4) {
        switch (C - c0) {
            case 1: latlong_backward_kernel<1><<<grid, LL_THREADS, 0, stream>>>(grad_cubemap, grad_panorama, d, c0); break;
            case 2: latlong_backward_kernel<2><<<grid, LL_THREADS, 0, stream>>>(grad_cubemap, grad_panorama, d, c0); break;
            case 3: latlong_backward_kernel<3><<<grid, LL_THREADS, 0, stream>>>(grad_cubemap, grad_panorama, d, c0); break;
            default: latlong_backward_kernel<4><<<grid, LL_THREADS, 0, stream>>>(grad_cubemap, grad_panorama, d, c0); break;
        }
        const cudaError_t e = launched();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace dirt
