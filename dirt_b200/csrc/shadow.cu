// shadow.cu -- shadow-map visibility (dirt_shadow_forward / dirt_shadow_backward, DESIGN.md §7.15): a percentage-closer
// lookup of a light-view map of (occupancy, depth) texels, the map that lighting.shadow_map rasterises.
//
// Per point p, with (x, y, z, w) = (p, 1) M for the light matrix M:
//   X = (x/w + 1) (0.5 SW),  Yd = (1 - y/w) (0.5 SH)   (the rasteriser's pixel rule, oracle/dirt_oracle.c S3, here
//   evaluated in double precision from the fp32 inputs),
//   c0 = floor(X - 0.5), fc = X - 0.5 - c0, and r0, fr the same of Yd,
//   V = sum_i sum_k a_i b_k s_ik / (2R+1)^2 over rows r0-R .. r0+R+1 and columns c0-R .. c0+R+1 (clamped into the map),
//   1-D weights (1 - f, 1, ..., 1, f), s_ik = 1 - o_ik step((z - z_ik - bias) / softness),
// step the logistic sigmoid for softness > 0 and the Heaviside step (step(0) = 0) for softness = 0.  A non-finite
// (x, y, z, w), w <= 0, or (X, Yd) outside [0, SW) x [0, SH) gives V = 1 and no gradient.
//
// One thread per point; a CTA holds 256 points of one item (blockIdx.x = chunk, blockIdx.y = item, looping past the grid
// limit), as the lighting kernels.  Texels are read as float2 through the read-only path.  The radius and softness > 0
// are template parameters, so the tap loops unroll.  The backward kernel recomputes the forward.  The light-matrix
// gradient is summed without atomics: per-CTA partial rows, then lighting.cu's fixed-order reduction, so it is
// bit-reproducible.  The map gradient is one float2 reduction per (tap, texel) and warp: the lanes of a warp whose tap
// hits the same texel add their (occupancy, depth) terms first (MATCH.ANY, common.cuh's agg_plan).
// Deterministic backward (dirt_shadow_backward_deterministic): the map gradient without float atomics.  The points are
// sorted by base texel with sort.cuh's radix sort, and each texel sums the terms of the (2R+2)^2 base segments that can
// reach it in a fixed order, in float64, rounded once; see the section below and DESIGN.md §7.15.
#include "../../include/dirt_b200.h"
#include "common.cuh"
#include "sort.cuh"

namespace dirt {

namespace {

constexpr int WARPS = LIGHT_THREADS / 32;
constexpr unsigned FULL = 0xffffffffu;

// The lookup of one point: its clip coordinates, validity, base texel and fractions.
struct ShadowPoint {
    float h[4];          // (x, y, z, w)
    float xn, yn;        // x / w, y / w
    float fr, fc;        // row and column fractions
    int r0, c0;          // base row and column (unclamped)
    bool valid;
};

// The coordinate chain runs in double precision: in fp32 the rounding of x/w alone moves X by several 1e-6 texels on a
// 2048-texel map, which shows in V through the weights 1 - f and f.  The taps and comparisons are fp32.
__device__ __forceinline__ ShadowPoint shadow_point(const float* __restrict__ M, const float p[3], int SH, int SW)
{
    ShadowPoint q;
    double h[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        h[c] = __fma_rn((double)p[2], (double)__ldg(M + 8 + c), __fma_rn((double)p[1], (double)__ldg(M + 4 + c),
                        __fma_rn((double)p[0], (double)__ldg(M + c), (double)__ldg(M + 12 + c))));
        q.h[c] = (float)h[c];
    }
    q.valid = isfinite(h[0]) && isfinite(h[1]) && isfinite(h[2]) && isfinite(h[3]) && h[3] > 0.0;
    const double xn = h[0] / h[3], yn = h[1] / h[3];
    q.xn = (float)xn;
    q.yn = (float)yn;
    const double X = (xn + 1.0) * (0.5 * SW), Yd = (1.0 - yn) * (0.5 * SH);
    q.valid = q.valid && X >= 0.0 && X < (double)SW && Yd >= 0.0 && Yd < (double)SH;
    if (!q.valid) {
        q.fr = q.fc = 0.f;
        q.r0 = q.c0 = 0;
        return q;
    }
    const double u = X - 0.5, v = Yd - 0.5;
    const double cf = floor(u), rf = floor(v);
    q.fc = (float)(u - cf);
    q.fr = (float)(v - rf);
    q.c0 = (int)cf;
    q.r0 = (int)rf;
    return q;
}

template <int R>
__device__ __forceinline__ float tap_weight(int i, float f)
{
    return i == 0 ? __fsub_rn(1.f, f) : (i == 2 * R + 1 ? f : 1.f);
}

__device__ __forceinline__ int clamp_to(int x, int n) { return x < 0 ? 0 : (x >= n ? n - 1 : x); }

// step((z - zj - bias) / softness) and, for SOFT, its derivative with respect to its argument's numerator
template <bool SOFT>
__device__ __forceinline__ float shadow_step(float d, float softness, float* dstep)
{
    if (!SOFT) {
        *dstep = 0.f;
        return d > 0.f ? 1.f : 0.f;
    }
    const float s = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-__fdiv_rn(d, softness))));
    *dstep = __fdiv_rn(__fmul_rn(s, __fsub_rn(1.f, s)), softness);
    return s;
}

__device__ __forceinline__ const float2* item_map(const ShadowArgs& a, long long b)
{
    return reinterpret_cast<const float2*>(a.map) + (a.per_item ? b * a.SH * (long long)a.SW : 0);
}

__device__ __forceinline__ const float* item_matrix(const ShadowArgs& a, long long b)
{
    return a.matrix + (a.per_item ? b * 16 : 0);
}

template <int R, bool SOFT>
__global__ void __launch_bounds__(LIGHT_THREADS) shadow_forward_kernel(ShadowArgs a)
{
    constexpr int T = 2 * R + 2;
    constexpr float INV_K = 1.f / (float)((2 * R + 1) * (2 * R + 1));
    __shared__ float stage[LIGHT_THREADS * 3];
    const int lane = threadIdx.x & 31;
    float* s = stage + (threadIdx.x & ~31) * 3;
    const long long v0 = (long long)blockIdx.x * LIGHT_THREADS + (threadIdx.x & ~31);
    if (v0 >= a.V) return;   // the whole warp
    const int n = (int)(a.V - v0 < 32 ? a.V - v0 : 32);
    for (long long b = blockIdx.y; b < a.B; b += gridDim.y) {
        const long long row0 = b * a.V + v0;
        float p[3];
        stage_load<3>(a.positions, a.sp, row0, n, s, lane, p);
        if (lane >= n) continue;
        const ShadowPoint q = shadow_point(item_matrix(a, b), p, a.SH, a.SW);
        float vis = 1.f;
        if (q.valid) {
            const float2* map = item_map(a, b);
            const float zb = __fsub_rn(q.h[2], a.bias);
            float acc = 0.f;
#pragma unroll
            for (int i = 0; i < T; ++i) {
                const long long rr = (long long)clamp_to(q.r0 - R + i, a.SH) * a.SW;
                float row = 0.f;
#pragma unroll
                for (int k = 0; k < T; ++k) {
                    const float2 t = __ldg(map + rr + clamp_to(q.c0 - R + k, a.SW));
                    float ds;
                    const float sv = __fsub_rn(1.f, __fmul_rn(t.x, shadow_step<SOFT>(__fsub_rn(zb, t.y), a.softness, &ds)));
                    row = __fmaf_rn(tap_weight<R>(k, q.fc), sv, row);
                }
                acc = __fmaf_rn(tap_weight<R>(i, q.fr), row, acc);
            }
            vis = __fmul_rn(acc, INV_K);
        }
        a.out[row0 + lane] = vis;
    }
}

// Sums the SHADOW_MATRIX values of every thread over the CTA in a fixed order (a butterfly in each warp, then the warps
// in order); thread j < SHADOW_MATRIX writes the j-th sum to dst[j].  Block-collective.
__device__ __forceinline__ void cta_matrix_partial(const float v[SHADOW_MATRIX], float* red, float* dst)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < SHADOW_MATRIX; ++j) {
        float x = v[j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(FULL, x, o);
        if (lane == 0) red[warp * SHADOW_MATRIX + j] = x;
    }
    __syncthreads();
    if (threadIdx.x < SHADOW_MATRIX) {
        float x = red[threadIdx.x];
#pragma unroll
        for (int w = 1; w < WARPS; ++w) x += red[w * SHADOW_MATRIX + threadIdx.x];
        dst[threadIdx.x] = x;
    }
    __syncthreads();
}

// (__maxnreg__ instead of __launch_bounds__: under the latter ptxas keeps two instances at 64 registers and spills)
template <int R, bool SOFT>
__global__ void __maxnreg__(96) shadow_backward_kernel(ShadowArgs a)
{
    constexpr int T = 2 * R + 2;
    constexpr float INV_K = 1.f / (float)((2 * R + 1) * (2 * R + 1));
    __shared__ float stage[LIGHT_THREADS * 3];
    __shared__ float red[WARPS * SHADOW_MATRIX];
    const int lane = threadIdx.x & 31;
    float* s = stage + (threadIdx.x & ~31) * 3;
    const long long v0 = (long long)blockIdx.x * LIGHT_THREADS + (threadIdx.x & ~31);
    const int n = v0 >= a.V ? 0 : (int)(a.V - v0 < 32 ? a.V - v0 : 32);   // warp-uniform; 0: the warp only helps reduce
    const bool live = lane < n;
    for (long long b = blockIdx.y; b < a.B; b += gridDim.y) {
        const long long row0 = b * a.V + v0, row = row0 + lane;
        const float* M = item_matrix(a, b);
        float p[3] = {0.f, 0.f, 0.f};
        if (n) stage_load<3>(a.positions, a.sp, row0, n, s, lane, p);
        ShadowPoint q = shadow_point(M, p, a.SH, a.SW);
        q.valid = q.valid && live;
        // an invalid point reads the texels around (0, 0) and adds nothing
        const float g = q.valid ? __fmul_rn(__ldg(a.grad_out + row), INV_K) : 0.f;
        // dV/dfr, dV/dfc, dV/dz, each times g / K
        float gfr = 0.f, gfc = 0.f, gz = 0.f;
        const float2* map = item_map(a, b);
        float2* gmap = reinterpret_cast<float2*>(a.g_map) + (a.per_item ? b * a.SH * (long long)a.SW : 0);
        const long long map_base = (a.per_item ? b * a.SH * (long long)a.SW : 0);
        const float zb = q.valid ? __fsub_rn(q.h[2], a.bias) : 0.f;   // a non-finite z would make 0 * step NaN
#pragma unroll 1
        for (int i = 0; i < T; ++i) {
            const int r = clamp_to(q.r0 - R + i, a.SH);
            const float wr = tap_weight<R>(i, q.fr);
            float row_b = 0.f, row_d = 0.f;   // sum_k b_k s_ik, s_i,last - s_i,0
#pragma unroll
            for (int k = 0; k < T; ++k) {
                const int c = clamp_to(q.c0 - R + k, a.SW);
                const float wc = tap_weight<R>(k, q.fc);
                const float2 t = __ldg(map + (long long)r * a.SW + c);
                float ds;
                const float st = shadow_step<SOFT>(__fsub_rn(zb, t.y), a.softness, &ds);
                const float sv = __fsub_rn(1.f, __fmul_rn(t.x, st));
                row_b = __fmaf_rn(wc, sv, row_b);
                if (k == 0) row_d = __fsub_rn(row_d, sv);
                if (k == T - 1) row_d = __fadd_rn(row_d, sv);
                const float w = __fmul_rn(wr, wc);
                if (SOFT) gz = __fmaf_rn(w, -__fmul_rn(t.x, ds), gz);
                if (a.g_map) {
                    // d V / d o = -w step, d V / d z_j = w o step' (softness > 0)
                    float v2[2] = {__fmul_rn(g, -__fmul_rn(w, st)), SOFT ? __fmul_rn(g, __fmul_rn(w, __fmul_rn(t.x, ds))) : 0.f};
                    const bool any = v2[0] != 0.f || v2[1] != 0.f;
                    const long long texel = (long long)r * a.SW + c;
                    // a lane with nothing to add takes a key no texel has
                    const unsigned long long key = any ? (unsigned long long)(map_base + texel) : ~0ull - lane;
                    const Agg ag = agg_plan(key, lane);
                    agg_sum<2>(ag, v2, lane);
                    if (any && __ffs(ag.peers) - 1 == lane) red_add_v2(reinterpret_cast<float*>(gmap + texel), v2[0], v2[1]);
                }
            }
            if (i == 0) gfr = __fsub_rn(gfr, row_b);
            if (i == T - 1) gfr = __fadd_rn(gfr, row_b);
            gfc = __fmaf_rn(wr, row_d, gfc);
        }
        // through X = (x/w + 1) (0.5 SW), Yd = (1 - y/w) (0.5 SH) to (x, y, z, w)
        float gh[4] = {0.f, 0.f, 0.f, 0.f};
        if (q.valid) {
            const float gxn = __fmul_rn(__fmul_rn(g, gfc), 0.5f * (float)a.SW);
            const float gyn = -__fmul_rn(__fmul_rn(g, gfr), 0.5f * (float)a.SH);
            gh[0] = __fdiv_rn(gxn, q.h[3]);
            gh[1] = __fdiv_rn(gyn, q.h[3]);
            gh[2] = __fmul_rn(g, gz);
            gh[3] = -__fdiv_rn(__fmaf_rn(gxn, q.xn, __fmul_rn(gyn, q.yn)), q.h[3]);
        }
        if (a.g_positions && n) {
            float gp[3];
#pragma unroll
            for (int j = 0; j < 3; ++j)
                gp[j] = __fmaf_rn(__ldg(M + 4 * j + 3), gh[3], __fmaf_rn(__ldg(M + 4 * j + 2), gh[2],
                                  __fmaf_rn(__ldg(M + 4 * j + 1), gh[1], __fmul_rn(__ldg(M + 4 * j), gh[0]))));
            stage_store<3>(a.g_positions, row0, n, s, lane, gp);
        }
        if (a.partial) {
            float v[SHADOW_MATRIX];
            const float ph[4] = {p[0], p[1], p[2], 1.f};
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int c = 0; c < 4; ++c) v[4 * j + c] = q.valid ? __fmul_rn(ph[j], gh[c]) : 0.f;
            cta_matrix_partial(v, red, a.partial + ((long long)b * a.chunks + blockIdx.x) * SHADOW_MATRIX);
        }
    }
}

// ---- deterministic backward ----------------------------------------------------------------------------------------
//
// A valid point's key is its base texel (r0, c0) on its map extended by one row and one column before the first
// (r0, c0 >= -1): (m (SH + 1) + r0 + 1) (SW + 1) + c0 + 1 for map m (the item's, or 0 when shared); an invalid point's
// is the sentinel, the number of keys.  The sort is stable, so each base segment lists its points by ascending id
// g = b V + n.  Texel (m, r, c) then sums, from +0.0 in float64, the fp32 terms of the default kernel (the same products,
// widened), in this order: tap row i = 0 .. 2R+1; every base row r0 whose tap row clamp(r0 - R + i) is r, ascending; tap
// column k = 0 .. 2R+1; every base column c0 whose tap column is c, ascending; the segment's points in order.  Off the
// map's edges exactly one base row (column) fits each tap; at an edge every base the clamp moves onto the edge does.
// One thread per texel, both channels, rounded once to fp32; every texel is written.
#ifndef DIRT_TEX_DET_GRID
#define DIRT_TEX_DET_GRID 8192   // texture.cu's cap of the deterministic passes' grids (one small-grid override for both)
#endif
constexpr unsigned DET_GRID = DIRT_TEX_DET_GRID;

__device__ __forceinline__ ShadowPoint point_of(const ShadowArgs& a, long long g, long long* b)
{
    *b = g / a.V;
    const float* pp = a.positions + g * a.sp;
    const float p[3] = {__ldg(pp), __ldg(pp + 1), __ldg(pp + 2)};
    return shadow_point(item_matrix(a, *b), p, a.SH, a.SW);
}

struct ShadowKey {
    ShadowArgs a;
    unsigned sentinel;
    __device__ __forceinline__ unsigned operator()(long long g) const
    {
        long long b;
        const ShadowPoint q = point_of(a, g, &b);
        if (!q.valid) return sentinel;
        const long long m = a.per_item ? b : 0;
        return (unsigned)((m * (a.SH + 1) + q.r0 + 1) * (long long)(a.SW + 1) + q.c0 + 1);
    }
};

// the base rows (columns) [*lo, *hi] whose tap i lands on row r of n rows
template <int R>
__device__ __forceinline__ void base_range(int r, int i, int n, int* lo, int* hi)
{
    *lo = r == 0 ? -1 : r + R - i;
    *hi = r == n - 1 ? n - 1 : r + R - i;
    if (*lo < -1) *lo = -1;
    if (*hi > n - 1) *hi = n - 1;
}

// (__maxnreg__ for the reason the backward kernel gives)
template <int R, bool SOFT>
__global__ void __maxnreg__(96) shadow_det_gather_kernel(ShadowArgs a, const int* __restrict__ ids,
                                                         const int* __restrict__ offsets)
{
    constexpr int T = 2 * R + 2;
    constexpr float INV_K = 1.f / (float)((2 * R + 1) * (2 * R + 1));
    const long long texels = (long long)a.SH * a.SW, total = (a.per_item ? a.B : 1) * texels;
    const long long stride = (long long)gridDim.x * LIGHT_THREADS;
    for (long long x = (long long)blockIdx.x * LIGHT_THREADS + threadIdx.x; x < total; x += stride) {
        const long long m = x / texels, rc = x - m * texels;
        const int r = (int)(rc / a.SW), c = (int)(rc - (long long)r * a.SW);
        const float2 t = __ldg(reinterpret_cast<const float2*>(a.map) + x);
        double so = 0.0, sd = 0.0;
#pragma unroll 1
        for (int i = 0; i < T; ++i) {
            int rlo, rhi;
            base_range<R>(r, i, a.SH, &rlo, &rhi);
            for (int r0 = rlo; r0 <= rhi; ++r0) {
#pragma unroll 1
                for (int k = 0; k < T; ++k) {
                    int clo, chi;
                    base_range<R>(c, k, a.SW, &clo, &chi);
                    for (int c0 = clo; c0 <= chi; ++c0) {
                        const long long key = (m * (a.SH + 1) + r0 + 1) * (long long)(a.SW + 1) + c0 + 1;
                        const int end = __ldg(offsets + key + 1);
                        for (int pos = __ldg(offsets + key); pos < end; ++pos) {
                            long long b;
                            const long long g = __ldg(ids + pos);
                            const ShadowPoint q = point_of(a, g, &b);
                            // the default kernel's terms: g / K times -w step and w o step'
                            const float gk = __fmul_rn(__ldg(a.grad_out + g), INV_K);
                            const float w = __fmul_rn(tap_weight<R>(i, q.fr), tap_weight<R>(k, q.fc));
                            float ds;
                            const float st = shadow_step<SOFT>(__fsub_rn(__fsub_rn(q.h[2], a.bias), t.y), a.softness, &ds);
                            const float vo = __fmul_rn(gk, -__fmul_rn(w, st));
                            so = __dadd_rn(so, (double)vo);
                            if (SOFT) sd = __dadd_rn(sd, (double)__fmul_rn(gk, __fmul_rn(w, __fmul_rn(t.x, ds))));
                        }
                    }
                }
            }
        }
        reinterpret_cast<float2*>(a.g_map)[x] = make_float2(__double2float_rn(so), __double2float_rn(sd));
    }
}

enum ShadowKernel { SHADOW_FORWARD, SHADOW_BACKWARD, SHADOW_GATHER };

template <int R, bool SOFT>
cudaError_t launch_rs(const ShadowArgs& a, ShadowKernel kind, const int* ids, const int* offsets, cudaStream_t stream)
{
    const dim3 grid = light_grid(a.chunks, a.B);
    if (kind == SHADOW_BACKWARD) {
        shadow_backward_kernel<R, SOFT><<<grid, LIGHT_THREADS, 0, stream>>>(a);
    } else if (kind == SHADOW_FORWARD) {
        shadow_forward_kernel<R, SOFT><<<grid, LIGHT_THREADS, 0, stream>>>(a);
    } else {
        const long long texels = (a.per_item ? a.B : 1) * (long long)a.SH * a.SW;
        const long long blocks = (texels + LIGHT_THREADS - 1) / LIGHT_THREADS;
        shadow_det_gather_kernel<R, SOFT><<<(unsigned)(blocks < DET_GRID ? blocks : DET_GRID), LIGHT_THREADS, 0, stream>>>(
            a, ids, offsets);
    }
    return launched();
}

template <int R>
cudaError_t launch_r(const ShadowArgs& a, ShadowKernel kind, const int* ids, const int* offsets, cudaStream_t stream)
{
    return a.softness > 0.f ? launch_rs<R, true>(a, kind, ids, offsets, stream)
                            : launch_rs<R, false>(a, kind, ids, offsets, stream);
}

cudaError_t launch_shadow(const ShadowArgs& a, ShadowKernel kind, cudaStream_t stream, const int* ids = nullptr,
                          const int* offsets = nullptr)
{
    switch (a.R) {
        case 0: return launch_r<0>(a, kind, ids, offsets, stream);
        case 1: return launch_r<1>(a, kind, ids, offsets, stream);
        case 2: return launch_r<2>(a, kind, ids, offsets, stream);
        default: return launch_r<3>(a, kind, ids, offsets, stream);
    }
}

}  // namespace

cudaError_t launch_shadow_forward(const ShadowArgs& a, cudaStream_t stream)
{
    if ((long long)a.B * a.V == 0) return cudaSuccess;
    return launch_shadow(a, SHADOW_FORWARD, stream);
}

cudaError_t launch_shadow_backward(const ShadowArgs& a, cudaStream_t stream)
{
    const long long items = a.per_item ? a.B : 1;
    cudaError_t e;
    if (a.g_map &&
        (e = cudaMemsetAsync(a.g_map, 0, sizeof(float) * 2 * (size_t)items * a.SH * a.SW, stream)) != cudaSuccess)
        return e;
    if (a.g_matrix && (long long)a.B * a.V == 0 &&
        (e = cudaMemsetAsync(a.g_matrix, 0, sizeof(float) * 16 * (size_t)items, stream)) != cudaSuccess)
        return e;
    if ((long long)a.B * a.V == 0 || (!a.g_positions && !a.g_matrix && !a.g_map)) return cudaSuccess;
    ShadowArgs b = a;
    if (!a.g_matrix) b.partial = nullptr;
    if ((e = launch_shadow(b, SHADOW_BACKWARD, stream)) != cudaSuccess) return e;
    if (!a.g_matrix) return cudaSuccess;
    return launch_partials_reduce(b.partial, a.g_matrix, SHADOW_MATRIX, a.per_item, a.chunks, a.B, stream);
}

ShadowDetScratch carve_shadow_det_scratch(void* base, const ShadowArgs& a)
{
    ShadowDetScratch s = {};
    char* p = static_cast<char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char* r = p ? p + off : nullptr;
        off = align_up(off + bytes, 256);
        return r;
    };
    const size_t n = (size_t)a.B * (size_t)a.V, tiles = (n + RS_TILE - 1) / RS_TILE;
    s.sentinel = (unsigned)(shadow_det_keys(a.B, a.per_item, a.SH, a.SW));
    for (int k = 0; k < 2; ++k) s.keys[k] = reinterpret_cast<unsigned*>(take(n * sizeof(unsigned)));
    for (int k = 0; k < 2; ++k) s.ids[k] = reinterpret_cast<int*>(take(n * sizeof(int)));
    s.offsets = reinterpret_cast<int*>(take(((size_t)s.sentinel + 2) * sizeof(int)));
    s.counts = reinterpret_cast<unsigned*>(take((size_t)RS_RADIX * tiles * sizeof(unsigned)));
    s.digit_total = reinterpret_cast<unsigned*>(take(RS_RADIX * sizeof(unsigned)));
    s.bytes = off;
    return s;
}

cudaError_t launch_shadow_backward_deterministic(const ShadowArgs& a, const ShadowDetScratch& s, cudaStream_t stream)
{
    // the position and matrix gradients have no atomics: the default kernel writes them
    if (!a.g_map || (long long)a.B * a.V == 0) return launch_shadow_backward(a, stream);
    cudaError_t e;
    ShadowArgs b = a;
    b.g_map = nullptr;
    if ((a.g_positions || a.g_matrix) && (e = launch_shadow_backward(b, stream)) != cudaSuccess) return e;
    int last;
    if ((e = sort_by_key(ShadowKey{a, s.sentinel}, (long long)a.B * a.V, s.sentinel, s.keys, s.ids, s.counts,
                         s.digit_total, stream, &last)) != cudaSuccess)
        return e;
    const long long bounds = ((long long)s.sentinel + 2 + RS_THREADS - 1) / RS_THREADS;
    tex_segment_bounds_kernel<<<(unsigned)(bounds < DET_GRID ? bounds : DET_GRID), RS_THREADS, 0, stream>>>(
        s.keys[last], (long long)a.B * a.V, s.sentinel, s.offsets);
    if ((e = launched()) != cudaSuccess) return e;
    return launch_shadow(a, SHADOW_GATHER, stream, s.ids[last], s.offsets);
}

}  // namespace dirt
