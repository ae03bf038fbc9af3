// ibl.cu -- image-based lighting (DESIGN.md §7.12): the texel table of a cube map's levels and the bounding cones of
// their 16 x 16 blocks, the GGX prefilter of levels 1 .. L-1 and its adjoint, the split-sum BRDF table, and the order-2
// SH projection of a cube map and its adjoint.  The lookup itself is §7.11's mipmapped cube-map lookup on the
// prefiltered levels (texture.cu).
//
// Prefilter: one CTA per 16 x 16 tile of output texels on one face of one level of one item, one thread per texel.
// The CTA tests every 16 x 16 block of source texels on any face against its tile, by their cones from the cone table
// widened by the lobe's support; the blocks that pass are listed in order, and each is staged in shared memory
// (direction and solid angle from the texel table, and the values) and read by every thread with broadcast loads.
// The staging is double-buffered with cp.async: the next block's copies run under the current block's arithmetic.
// The adjoint is the same loop with the roles of source and output swapped: a gather, with no atomics.
#include "../../include/dirt_b200.h"
#include "common.cuh"

#include <cmath>
#include <type_traits>

namespace dirt {

namespace {

constexpr int IBL_TILE = 16;                      // tile and staged block edge
constexpr int IBL_THREADS = IBL_TILE * IBL_TILE;  // one thread per tile texel, one staged texel per thread
// grid caps (grid-stride loops beyond them); a build may lower them to test those loops
#ifndef DIRT_IBL_MAX_ITEMS
#define DIRT_IBL_MAX_ITEMS 65535
#endif
#ifndef DIRT_IBL_MAX_BLOCKS
#define DIRT_IBL_MAX_BLOCKS 65536
#endif
constexpr int IBL_MAX_ITEMS = DIRT_IBL_MAX_ITEMS;     // gridDim.y of the prefilter, its adjoint and the SH partial sums
constexpr long long IBL_MAX_BLOCKS = DIRT_IBL_MAX_BLOCKS;
// 1: the staged blocks are double-buffered with cp.async; 0: loaded through registers, one block at a time (the
// alternative it was measured against, DESIGN.md §7.12)
#ifndef DIRT_IBL_CP_ASYNC
#define DIRT_IBL_CP_ASYNC 1
#endif
constexpr bool IBL_CP_ASYNC = DIRT_IBL_CP_ASYNC != 0;
constexpr unsigned IBL_FULL = 0xffffffffu;
constexpr float IBL_CONE_SLACK = 4e-3f;           // radians added to the cone test: fp32 acos near 1 is good to ~4e-4
constexpr double IBL_MIN_ROUGHNESS = 0.045;       // GGX_MIN_ROUGHNESS of lighting.py, in float64

// One thread per texel of every level: (direction, solid angle).  sc = (2c+1)/S_k - 1 and tc = (2r+1)/S_k - 1 in
// fp32, the face table, then x / sqrt(fma(z, z, fma(y, y, x*x))) for each component, each operation rounded in that
// order; the solid angle by the corner formula in float64, rounded once.
__global__ void __launch_bounds__(IBL_THREADS) ggx_texel_table_kernel(float4* __restrict__ table, IblLevels p)
{
    const long long n = p.table[p.L], stride = (long long)gridDim.x * IBL_THREADS;
    for (long long e = (long long)blockIdx.x * IBL_THREADS + threadIdx.x; e < n; e += stride) {
        int k = 0;
        while (e >= p.table[k + 1]) ++k;
        const int Sk = p.S >> k;
        const long long x = e - p.table[k];
        const int f = (int)(x / ((long long)Sk * Sk)), rc = (int)(x - (long long)f * Sk * Sk), r = rc / Sk, c = rc - r * Sk;
        const float Sf = (float)Sk;
        const float sc = __fsub_rn(__fdiv_rn((float)(2 * c + 1), Sf), 1.0f), tc = __fsub_rn(__fdiv_rn((float)(2 * r + 1), Sf), 1.0f);
        float dx, dy, dz;
        face_point(f, sc, tc, dx, dy, dz);
        const float len = __fsqrt_rn(__fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx))));
        const double u0 = 2.0 * c / Sk - 1.0, u1 = 2.0 * (c + 1) / Sk - 1.0, v0 = 2.0 * r / Sk - 1.0, v1 = 2.0 * (r + 1) / Sk - 1.0;
        auto F = [](double u, double v) { return atan2(u * v, sqrt(u * u + v * v + 1.0)); };
        const double omega = F(u1, v1) - F(u0, v1) - F(u1, v0) + F(u0, v0);
        table[e] = make_float4(__fdiv_rn(dx, len), __fdiv_rn(dy, len), __fdiv_rn(dz, len), (float)omega);
    }
}

// The cone around texels [r0, r1) x [c0, c1) of face f at S per edge, texel edges included: its axis through the
// rectangle's centre and the half-angle to its farthest corner, float64.  The rectangle's directions lie inside it
// (its image on the sphere is convex and within 90 degrees of the axis).
struct Cone {
    float x, y, z, theta;
};

__device__ __forceinline__ Cone rect_cone(int f, int S, int r0, int r1, int c0, int c1)
{
    const float u0 = 2.f * c0 / S - 1.f, u1 = 2.f * c1 / S - 1.f, v0 = 2.f * r0 / S - 1.f, v1 = 2.f * r1 / S - 1.f;
    Cone a;
    face_point(f, 0.5f * (u0 + u1), 0.5f * (v0 + v1), a.x, a.y, a.z);
    const float il = rsqrtf(a.x * a.x + a.y * a.y + a.z * a.z);
    a.x *= il;
    a.y *= il;
    a.z *= il;
    float cmin = 1.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        float x, y, z;
        face_point(f, q & 1 ? u1 : u0, q & 2 ? v1 : v0, x, y, z);
        cmin = fminf(cmin, (a.x * x + a.y * y + a.z * z) * rsqrtf(x * x + y * y + z * z));
    }
    a.theta = acosf(fmaxf(-1.f, fminf(1.f, cmin)));
    return a;
}

// In the lobe's reach: the angle between the axes at most both half-angles plus the support's (and the slack)
__device__ __forceinline__ bool cones_meet(const Cone& a, const Cone& b, float reach)
{
    const float c = fmaxf(-1.f, fminf(1.f, a.x * b.x + a.y * b.y + a.z * b.z));
    return acosf(c) <= a.theta + b.theta + reach + IBL_CONE_SLACK;
}

// One thread per 16 x 16 block of every level's six faces: its cone, (axis, half-angle), shared by every CTA and item
__global__ void __launch_bounds__(IBL_THREADS) ggx_cone_table_kernel(float4* __restrict__ cones, IblLevels p)
{
    const long long n = p.cone[p.L], stride = (long long)gridDim.x * IBL_THREADS;
    for (long long e = (long long)blockIdx.x * IBL_THREADS + threadIdx.x; e < n; e += stride) {
        int k = 0;
        while (e >= p.cone[k + 1]) ++k;
        const int Sk = p.S >> k, nb = (Sk + IBL_TILE - 1) / IBL_TILE;
        const int x = (int)(e - p.cone[k]), f = x / (nb * nb), b = x - f * nb * nb;
        const int r0 = (b / nb) * IBL_TILE, c0 = (b % nb) * IBL_TILE;
        const Cone a = rect_cone(f, Sk, r0, min(r0 + IBL_TILE, Sk), c0, min(c0 + IBL_TILE, Sk));
        cones[e] = make_float4(a.x, a.y, a.z, a.theta);
    }
}

__device__ __forceinline__ Cone cone_of(const float4& v) { return Cone{v.x, v.y, v.z, v.w}; }

// cp.async of 16 / 4 bytes into shared memory, zero-filled when !full (src is then not read)
__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool full)
{
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(src), "r"(full ? 16 : 0));
}

__device__ __forceinline__ void cp_async4(void* dst, const void* src, bool full)
{
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(d), "l"(src), "r"(full ? 4 : 0));
}

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }

template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// Ordered compaction of the CTA's candidates: the kept values, in thread order, to list[0 ..); returns their number
__device__ __forceinline__ int compact(bool keep, int value, int* list, int* warp_counts)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned m = __ballot_sync(IBL_FULL, keep);
    if (lane == 0) warp_counts[warp] = __popc(m);
    __syncthreads();
    int base = 0, total = 0;
#pragma unroll
    for (int w = 0; w < IBL_THREADS / 32; ++w) {
        base += w < warp ? warp_counts[w] : 0;
        total += warp_counts[w];
    }
    if (keep) list[base + __popc(m & ((1u << lane) - 1u))] = value;
    __syncthreads();
    return total;
}

// the work item of CTA x: level (from the prefix `first`), face and tile
struct IblTile {
    int k, f, r0, c0;
};

__device__ __forceinline__ IblTile tile_of(const int* first, const int* level, int n, int S, int x)
{
    int w = 0;
    while (w + 1 < n && x >= first[w + 1]) ++w;
    IblTile t;
    t.k = level[w];
    const int nb = ((S >> t.k) + IBL_TILE - 1) / IBL_TILE;
    const int y = x - first[w];
    t.f = y / (nb * nb);
    const int b = y - t.f * nb * nb;
    t.r0 = (b / nb) * IBL_TILE;
    t.c0 = (b % nb) * IBL_TILE;
    return t;
}

// c = fma(r.z, l.z, fma(r.y, l.y, r.x * l.x)): symmetric in r and l, so the adjoint sees the forward's pairs
__device__ __forceinline__ float pair_cos(float rx, float ry, float rz, const float4& l)
{
    return __fmaf_rn(rz, l.z, __fmaf_rn(ry, l.y, __fmul_rn(rx, l.x)));
}

// Level k >= 1 (tile of the CTA) from source level s = min(k, s*): P = sum_j w_j src_j / W, w_j = D(c) c Omega_j over the
// source texels with c > 0 and c >= c_k, summed in the order of the listed blocks and, inside one, of the texels
// (row-major).  The sums leave out D's constant alpha2 / pi, which cancels in P; W is written with it.  NV channels
// c0 .. c0+NV-1 per launch; the first launch (write_w) also writes W.
template <int NV>
__global__ void __launch_bounds__(IBL_THREADS) ggx_prefilter_kernel(const float* __restrict__ cubemap,
                                                                    const float* __restrict__ box,
                                                                    const float4* __restrict__ table,
                                                                    const float4* __restrict__ cones,
                                                                    float* __restrict__ levels, float* __restrict__ W,
                                                                    IblLevels p, int c0, bool write_w)
{
    __shared__ float4 sdir[2][IBL_THREADS];
    __shared__ float sval[2][NV * IBL_THREADS];
    __shared__ int list[IBL_THREADS];
    __shared__ int warp_counts[IBL_THREADS / 32];
    const int tid = threadIdx.x, C = p.C;
    const IblTile t = tile_of(p.first, p.level, p.works, p.S, blockIdx.x);
    const int k = t.k, Sk = p.S >> k, s = k < p.ss ? k : p.ss, Ss = p.S >> s, nb = (Ss + IBL_TILE - 1) / IBL_TILE;
    const int nbk = (Sk + IBL_TILE - 1) / IBL_TILE;
    const int r = t.r0 + (tid >> 4), c = t.c0 + (tid & 15);
    const bool valid = r < Sk && c < Sk;
    const float4 me = valid ? table[p.table[k] + ((long long)t.f * Sk + r) * Sk + c] : make_float4(0.f, 0.f, 0.f, 0.f);
    const Cone tc = cone_of(cones[p.cone[k] + ((long long)t.f * nbk + t.r0 / IBL_TILE) * nbk + t.c0 / IBL_TILE]);
    const float alpha2 = p.alpha2[k], ck = p.ck[k], half = p.half[k], dn = p.dn[k];
    const float reach = acosf(ck);
    const long long face_texels = (long long)Ss * Ss;
    const float* src = s == 0 ? cubemap : box + 6ll * p.TB * p.pyr[s] * C;
    const float4* stab = table + p.table[s];
    const int candidates = 6 * nb * nb;
    for (int tb = blockIdx.y; tb < p.TB; tb += gridDim.y) {
        const float* item = src + tb * 6ll * face_texels * C + c0;
        float W_acc = 0.f, acc[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) acc[j] = 0.f;
        // this thread's texel of listed block cb into buffer b
        auto stage = [&](int cb, int b) {
            const int fs = cb / (nb * nb), bb = cb - fs * nb * nb;
            const int rr = (bb / nb) * IBL_TILE + (tid >> 4), cc = (bb % nb) * IBL_TILE + (tid & 15);
            const bool in = rr < Ss && cc < Ss;
            const long long x = in ? ((long long)fs * Ss + rr) * Ss + cc : 0;
            if constexpr (IBL_CP_ASYNC) {
                cp_async16(&sdir[b][tid], stab + x, in);
#pragma unroll
                for (int j = 0; j < NV; ++j) cp_async4(&sval[b][j * IBL_THREADS + tid], item + x * C + j, in);
            } else {
                sdir[b][tid] = in ? stab[x] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int j = 0; j < NV; ++j) sval[b][j * IBL_THREADS + tid] = in ? __ldg(item + x * C + j) : 0.f;
            }
        };
        auto consume = [&](int b) {
            if (!valid) return;
#pragma unroll 4
            for (int q = 0; q < IBL_THREADS; ++q) {
                const float4 l = sdir[b][q];
                const float cs = pair_cos(me.x, me.y, me.z, l);
                if (cs > 0.f && cs >= ck) {
                    const float kk = __fmaf_rn(1.0f - cs, half, alpha2);
                    const float w = __fdividef(cs * l.w, kk * kk);
                    W_acc += w;
#pragma unroll
                    for (int j = 0; j < NV; ++j) acc[j] = __fmaf_rn(w, sval[b][j * IBL_THREADS + q], acc[j]);
                }
            }
        };
        for (int b0 = 0; b0 < candidates; b0 += IBL_THREADS) {
            const int cand = b0 + tid;
            const bool keep = cand < candidates && cones_meet(tc, cone_of(cones[p.cone[s] + cand]), reach);
            const int n = compact(keep, cand, list, warp_counts);
            if constexpr (IBL_CP_ASYNC) {
                if (n > 0) {
                    stage(list[0], 0);
                    cp_async_commit();
                }
                for (int i = 0; i < n; ++i) {
                    if (i + 1 < n) {
                        stage(list[i + 1], (i + 1) & 1);
                        cp_async_commit();
                        cp_async_wait<1>();
                    } else {
                        cp_async_wait<0>();
                    }
                    __syncthreads();
                    consume(i & 1);
                    __syncthreads();
                }
            } else {
                for (int i = 0; i < n; ++i) {
                    stage(list[i], 0);
                    __syncthreads();
                    consume(0);
                    __syncthreads();
                }
            }
        }
        if (valid) {
            const long long x = ((long long)t.f * Sk + r) * Sk + c;
            if (write_w && tb == 0) W[6ll * p.pyr[k] + x] = __fmul_rn(W_acc, dn);
            float* o = levels + (6ll * p.TB * p.pyr[k] + tb * 6ll * Sk * Sk + x) * C + c0;
#pragma unroll
            for (int j = 0; j < NV; ++j) o[j] = __fdiv_rn(acc[j], W_acc);
        }
    }
}

// The prefilter's adjoint for the source texels of the CTA's tile on level s: grad_src_j = sum over the output levels
// k with min(k, s*) = s, in level order, of Omega_j * sum_r D_k(c) c g_k(r) / W_k(r) over the forward's pairs.  Written
// to out's level s (s >= 1), or added to grad_cubemap (s = 0).  Staged per output texel: direction, g_k and W_k, then
// g_k / W_k in place by the thread that staged it.
template <int NV>
__global__ void __launch_bounds__(IBL_THREADS) ggx_prefilter_adjoint_kernel(const float* __restrict__ level_grad,
                                                                            const float* __restrict__ W,
                                                                            const float4* __restrict__ table,
                                                                            const float4* __restrict__ cones,
                                                                            float* __restrict__ out,
                                                                            float* __restrict__ grad_cubemap, IblLevels p,
                                                                            int c0)
{
    __shared__ float4 sdir[2][IBL_THREADS];
    __shared__ float sval[2][NV * IBL_THREADS];
    __shared__ float sw[2][IBL_THREADS];
    __shared__ int list[IBL_THREADS];
    __shared__ int warp_counts[IBL_THREADS / 32];
    const int tid = threadIdx.x, C = p.C;
    const IblTile t = tile_of(p.first, p.level, p.works, p.S, blockIdx.x);
    const int s = t.k, Ss = p.S >> s, nbs = (Ss + IBL_TILE - 1) / IBL_TILE;
    const int r = t.r0 + (tid >> 4), c = t.c0 + (tid & 15);
    const bool valid = r < Ss && c < Ss;
    const float4 me = valid ? table[p.table[s] + ((long long)t.f * Ss + r) * Ss + c] : make_float4(0.f, 0.f, 0.f, 0.f);
    const Cone tc = cone_of(cones[p.cone[s] + ((long long)t.f * nbs + t.r0 / IBL_TILE) * nbs + t.c0 / IBL_TILE]);
    const int k_first = s == p.ss ? (s > 0 ? s : 1) : s, k_last = s == p.ss ? p.L - 1 : s;
    for (int tb = blockIdx.y; tb < p.TB; tb += gridDim.y) {
        float total[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) total[j] = 0.f;
        for (int k = k_first; k <= k_last; ++k) {
            const int Sk = p.S >> k, nb = (Sk + IBL_TILE - 1) / IBL_TILE, candidates = 6 * nb * nb;
            const float alpha2 = p.alpha2[k], ck = p.ck[k], half = p.half[k], dn = p.dn[k];
            const float reach = acosf(ck);
            const float* g = level_grad + (6ll * p.TB * p.pyr[k] + tb * 6ll * Sk * Sk) * C + c0;
            const float* Wk = W + 6ll * p.pyr[k];
            const float4* ktab = table + p.table[k];
            float acc[NV];
#pragma unroll
            for (int j = 0; j < NV; ++j) acc[j] = 0.f;
            auto stage = [&](int cb, int b) {
                const int fo = cb / (nb * nb), bb = cb - fo * nb * nb;
                const int rr = (bb / nb) * IBL_TILE + (tid >> 4), cc = (bb % nb) * IBL_TILE + (tid & 15);
                const bool in = rr < Sk && cc < Sk;
                const long long x = in ? ((long long)fo * Sk + rr) * Sk + cc : 0;
                if constexpr (IBL_CP_ASYNC) {
                    cp_async16(&sdir[b][tid], ktab + x, in);
#pragma unroll
                    for (int j = 0; j < NV; ++j) cp_async4(&sval[b][j * IBL_THREADS + tid], g + x * C + j, in);
                    cp_async4(&sw[b][tid], Wk + x, in);
                } else {
                    sdir[b][tid] = in ? ktab[x] : make_float4(0.f, 0.f, 0.f, 0.f);
                    const float wr = in ? __ldg(Wk + x) : 0.f;
#pragma unroll
                    for (int j = 0; j < NV; ++j)
                        sval[b][j * IBL_THREADS + tid] = in ? __fdividef(__ldg(g + x * C + j), wr) : 0.f;
                }
            };
            // g / W in place, by the thread whose copies these are (cp.async only)
            auto finish = [&](int b) {
                const float wr = sw[b][tid];
#pragma unroll
                for (int j = 0; j < NV; ++j)
                    sval[b][j * IBL_THREADS + tid] = wr != 0.f ? __fdividef(sval[b][j * IBL_THREADS + tid], wr) : 0.f;
            };
            auto consume = [&](int b) {
                if (!valid) return;
#pragma unroll 4
                for (int q = 0; q < IBL_THREADS; ++q) {
                    const float4 l = sdir[b][q];
                    const float cs = pair_cos(l.x, l.y, l.z, me);
                    if (cs > 0.f && cs >= ck) {
                        const float kk = __fmaf_rn(1.0f - cs, half, alpha2);
                        const float w = __fdividef(cs * dn, kk * kk);
#pragma unroll
                        for (int j = 0; j < NV; ++j) acc[j] = __fmaf_rn(w, sval[b][j * IBL_THREADS + q], acc[j]);
                    }
                }
            };
            for (int b0 = 0; b0 < candidates; b0 += IBL_THREADS) {
                const int cand = b0 + tid;
                const bool keep = cand < candidates && cones_meet(tc, cone_of(cones[p.cone[k] + cand]), reach);
                const int n = compact(keep, cand, list, warp_counts);
                if constexpr (IBL_CP_ASYNC) {
                    if (n > 0) {
                        stage(list[0], 0);
                        cp_async_commit();
                    }
                    for (int i = 0; i < n; ++i) {
                        if (i + 1 < n) {
                            stage(list[i + 1], (i + 1) & 1);
                            cp_async_commit();
                            cp_async_wait<1>();
                        } else {
                            cp_async_wait<0>();
                        }
                        finish(i & 1);
                        __syncthreads();
                        consume(i & 1);
                        __syncthreads();
                    }
                } else {
                    for (int i = 0; i < n; ++i) {
                        stage(list[i], 0);
                        __syncthreads();
                        consume(0);
                        __syncthreads();
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < NV; ++j) total[j] = __fadd_rn(total[j], __fmul_rn(me.w, acc[j]));
        }
        if (valid) {
            const long long x = tb * 6ll * Ss * Ss + ((long long)t.f * Ss + r) * Ss + c;
            if (s == 0) {
                float* o = grad_cubemap + x * C + c0;
#pragma unroll
                for (int j = 0; j < NV; ++j) o[j] = __fadd_rn(o[j], total[j]);
            } else {
                float* o = out + (6ll * p.TB * p.pyr[s] + x) * C + c0;
#pragma unroll
                for (int j = 0; j < NV; ++j) o[j] = total[j];
            }
        }
    }
}

// One thread per node (i, j) of the N x N table, n.v = (i + 0.5) / N and roughness (j + 0.5) / N: (A, B) by a midpoint
// rule over the GGX half-vector distribution, in float64.  h: cos(theta_h)^2 = (1 - u) / (1 + (alpha2 - 1) u) at
// u = 1 - t^2, t = (a + 0.5) / BRDF_U (the substitution makes the integrand's 1 / sqrt(1 - u) at grazing half-vectors
// smooth), phi = 2 pi (b + 0.5) / BRDF_PHI (cos by cospi); l = 2 (v.h) h - v; each sample adds Vis (n.l) 4 (v.h) / (n.h) 2t times
// (1 - F_c) to A and F_c to B where n.l > 0 and v.h > 0.
constexpr int BRDF_U = 1024, BRDF_PHI = 64;

__global__ void __launch_bounds__(128) ggx_brdf_table_kernel(float* __restrict__ table, int N)
{
    const int e = blockIdx.x * 128 + threadIdx.x;
    if (e >= N * N) return;
    const int i = e / N, j = e - i * N;
    const double nv = (i + 0.5) / N, rough = (j + 0.5) / N;
    const double a = fmax(rough, IBL_MIN_ROUGHNESS), alpha2 = (a * a) * (a * a);
    const double vx = sqrt(1.0 - nv * nv), vz = nv;
    const double sv = sqrt(nv * nv * (1.0 - alpha2) + alpha2);
    double A = 0.0, B = 0.0;
    for (int u = 0; u < BRDF_U; ++u) {
        const double tu = (u + 0.5) / BRDF_U, x = 1.0 - tu * tu;
        const double ch = sqrt((1.0 - x) / (1.0 + (alpha2 - 1.0) * x)), sh = sqrt(fmax(0.0, 1.0 - ch * ch));
        for (int b = 0; b < BRDF_PHI; ++b) {
            const double hx = sh * cospi(2.0 * (b + 0.5) / BRDF_PHI), hz = ch;
            const double vh = vx * hx + vz * hz;
            const double nl = 2.0 * vh * hz - vz;
            if (nl <= 0.0 || vh <= 0.0) continue;
            const double vis = 0.5 / (nl * sv + nv * sqrt(nl * nl * (1.0 - alpha2) + alpha2));
            const double g = vis * nl * 4.0 * vh / ch * (2.0 * tu);
            const double m = 1.0 - vh, fc = (m * m) * (m * m) * m;
            A += (1.0 - fc) * g;
            B += fc * g;
        }
    }
    const double n = (double)BRDF_U * BRDF_PHI;
    table[2 * e] = (float)(A / n);
    table[2 * e + 1] = (float)(B / n);
}

// ---- order-2 SH projection of a cube map: L_k = sum_j L(l_j) Y_k(l_j) Omega_j over level 0's texel table ----

constexpr int CUBE_SH_CHUNK = 4096;   // texels per partial sum

// lighting.py's _sh_basis, float64
__device__ __forceinline__ void sh_basis(double x, double y, double z, double Y[9])
{
    Y[0] = 0.28209479177387814;
    Y[1] = 0.4886025119029199 * y;
    Y[2] = 0.4886025119029199 * z;
    Y[3] = 0.4886025119029199 * x;
    Y[4] = 1.0925484305920792 * x * y;
    Y[5] = 1.0925484305920792 * y * z;
    Y[6] = 0.31539156525252005 * (3 * z * z - 1);
    Y[7] = 1.0925484305920792 * x * z;
    Y[8] = 0.5462742152960396 * (x * x - y * y);
}

// Per item and chunk of CUBE_SH_CHUNK texels, per channel: the chunk's nine sums in float64, each thread over its texels in
// order, then a fixed tree across the CTA; partial [TB, chunks, 9, C]
__global__ void __launch_bounds__(IBL_THREADS) sh_project_partial_kernel(const float* __restrict__ cubemap,
                                                                         const float4* __restrict__ table,
                                                                         double* __restrict__ partial, long long n,
                                                                         int TB, int C, int chunks)
{
    __shared__ double red[9][IBL_THREADS];
    const int tid = threadIdx.x;
    for (int tb = blockIdx.y; tb < TB; tb += gridDim.y) {
        for (int ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
            const long long j0 = (long long)ch * CUBE_SH_CHUNK, j1 = j0 + CUBE_SH_CHUNK < n ? j0 + CUBE_SH_CHUNK : n;
            for (int c = 0; c < C; ++c) {
                double acc[9];
#pragma unroll
                for (int q = 0; q < 9; ++q) acc[q] = 0.0;
                for (long long j = j0 + tid; j < j1; j += IBL_THREADS) {
                    const float4 e = table[j];
                    const double v = (double)__ldg(cubemap + ((long long)tb * n + j) * C + c) * (double)e.w;
                    double Y[9];
                    sh_basis(e.x, e.y, e.z, Y);
#pragma unroll
                    for (int q = 0; q < 9; ++q) acc[q] += v * Y[q];
                }
#pragma unroll
                for (int q = 0; q < 9; ++q) red[q][tid] = acc[q];
                __syncthreads();
                for (int h = IBL_THREADS / 2; h > 0; h >>= 1) {
                    if (tid < h)
#pragma unroll
                        for (int q = 0; q < 9; ++q) red[q][tid] += red[q][tid + h];
                    __syncthreads();
                }
                if (tid < 9) partial[(((long long)tb * chunks + ch) * 9 + tid) * C + c] = red[tid][0];
                __syncthreads();
            }
        }
    }
}

// One thread per (item, k, channel): the chunks' sums in chunk order, rounded once
__global__ void __launch_bounds__(IBL_THREADS) sh_project_final_kernel(const double* __restrict__ partial,
                                                                       float* __restrict__ out, int TB, int C, int chunks)
{
    const long long n = (long long)TB * 9 * C, stride = (long long)gridDim.x * IBL_THREADS;
    for (long long e = (long long)blockIdx.x * IBL_THREADS + threadIdx.x; e < n; e += stride) {
        const long long tb = e / (9 * C), kc = e - tb * 9 * C;
        double sum = 0.0;
        for (int ch = 0; ch < chunks; ++ch) sum += partial[((long long)tb * chunks + ch) * 9 * C + kc];
        out[e] = (float)sum;
    }
}

// The adjoint, one thread per cube-map element: Omega_j sum_k Y_k(l_j) g_k, float64 rounded once
__global__ void __launch_bounds__(IBL_THREADS) sh_project_backward_kernel(const float4* __restrict__ table,
                                                                          const float* __restrict__ grad_coeffs,
                                                                          float* __restrict__ grad_cubemap, long long n,
                                                                          int TB, int C)
{
    const long long total = (long long)TB * n * C, stride = (long long)gridDim.x * IBL_THREADS;
    for (long long e = (long long)blockIdx.x * IBL_THREADS + threadIdx.x; e < total; e += stride) {
        const long long x = e / C, tb = x / n, j = x - tb * n;
        const int c = (int)(e - x * C);
        const float4 t = table[j];
        double Y[9];
        sh_basis(t.x, t.y, t.z, Y);
        double sum = 0.0;
#pragma unroll
        for (int q = 0; q < 9; ++q) sum += Y[q] * (double)__ldg(grad_coeffs + (tb * 9 + q) * C + c);
        grad_cubemap[e] = (float)(sum * (double)t.w);
    }
}

inline unsigned ibl_blocks(long long work)
{
    const long long b = (work + IBL_THREADS - 1) / IBL_THREADS;
    return (unsigned)(b < IBL_MAX_BLOCKS ? (b > 0 ? b : 1) : IBL_MAX_BLOCKS);
}

template <typename F>
cudaError_t with_nv(int nv, F f)
{
    switch (nv) {
        case 1: return f(std::integral_constant<int, 1>{});
        case 2: return f(std::integral_constant<int, 2>{});
        case 3: return f(std::integral_constant<int, 3>{});
        default: return f(std::integral_constant<int, 4>{});
    }
}

// the work list: CTA tiles of the given levels, in order
void set_works(IblLevels& p, const int* levels, int n)
{
    p.works = n;
    int x = 0;
    for (int w = 0; w < n; ++w) {
        p.level[w] = levels[w];
        p.first[w] = x;
        const int nb = ((p.S >> levels[w]) + IBL_TILE - 1) / IBL_TILE;
        x += 6 * nb * nb;
    }
    p.first[n] = x;
}

}  // namespace

// d: the cube map's dims (TW = S + 2)
IblLevels ibl_levels(const TexDims& d)
{
    IblLevels p = {};
    p.S = d.TW - 2;
    p.TB = d.TB;
    p.C = d.C;
    p.L = mip_levels(p.S, p.S);
    p.ss = 0;
    for (int k = 0; k < p.L; ++k)
        if ((p.S >> k) >= 16) p.ss = k;
    const long long texels = (long long)p.S * p.S;
    for (int k = 0; k <= p.L; ++k) {
        p.table[k] = k == 0 ? 0 : p.table[k - 1] + 6 * (texels >> (2 * (k - 1)));
        p.pyr[k] = k == 0 ? 0 : (texels - (texels >> (2 * (k - 1)))) / 3;
        const long long nb = k == 0 ? 0 : (((p.S >> (k - 1)) + IBL_TILE - 1) / IBL_TILE);
        p.cone[k] = k == 0 ? 0 : p.cone[k - 1] + 6 * nb * nb;
    }
    for (int k = 1; k < p.L; ++k) {
        const double r = (double)k / (p.L - 1), a = r > IBL_MIN_ROUGHNESS ? r : IBL_MIN_ROUGHNESS;
        const double alpha2 = (a * a) * (a * a);
        const double ck = alpha2 >= 1.0 ? 0.0 : 1.0 - 2.0 * (std::sqrt(1000.0) - 1.0) * alpha2 / (1.0 - alpha2);
        p.alpha2[k] = (float)alpha2;
        p.ck[k] = (float)(ck > 0.0 ? ck : 0.0);
        p.half[k] = (float)((1.0 - alpha2) * 0.5);
        p.dn[k] = (float)(alpha2 / M_PI);
    }
    return p;
}

GgxLayout ggx_layout(const TexDims& d)
{
    const IblLevels p = ibl_levels(d);
    GgxLayout g;
    g.levels = (long long)cubemap_mip_atlas_texels(d) * d.C;
    g.weights = g.levels + 6ll * d.TB * p.pyr[p.L] * d.C;
    g.table = (g.weights + 6ll * p.pyr[p.L] + 3) / 4 * 4;
    g.cones = g.table + 4 * p.table[p.L];
    g.floats = g.cones + 4 * p.cone[p.L];
    return g;
}

cudaError_t launch_ggx_prefilter(const float* cubemap, float* atlas, const TexDims& d, cudaStream_t stream)
{
    const IblLevels p0 = ibl_levels(d);
    if (p0.L == 1 || d.TB == 0) return cudaSuccess;
    const GgxLayout g = ggx_layout(d);
    float4* table = reinterpret_cast<float4*>(atlas + g.table);
    cudaError_t e;
    // the box pyramid of the 6 * TB faces in level 0's slot of the mip atlas, as texture.cu's mipmapped lookup builds it
    TexDims pd = d;
    pd.TB = 6 * d.TB;
    pd.TH = pd.TW = p0.S;
    pd.texels = (long long)p0.S * p0.S;
    pd.total = 0;
    pd.mode = DIRT_TEXTURE_BILINEAR;
    if (p0.ss > 0 && (e = launch_texture_mip_build(cubemap, atlas, pd, stream)) != cudaSuccess) return e;
    float4* cones = reinterpret_cast<float4*>(atlas + g.cones);
    ggx_texel_table_kernel<<<ibl_blocks(p0.table[p0.L]), IBL_THREADS, 0, stream>>>(table, p0);
    if ((e = launched()) != cudaSuccess) return e;
    ggx_cone_table_kernel<<<ibl_blocks(p0.cone[p0.L]), IBL_THREADS, 0, stream>>>(cones, p0);
    if ((e = launched()) != cudaSuccess) return e;
    IblLevels p = p0;
    int levels[MIP_MAX_LEVELS];
    for (int k = 1; k < p.L; ++k) levels[k - 1] = k;
    set_works(p, levels, p.L - 1);
    const dim3 grid(p.first[p.works], d.TB < IBL_MAX_ITEMS ? d.TB : IBL_MAX_ITEMS);
    for (int c0 = 0; c0 < d.C; c0 += 4) {
        e = with_nv(d.C - c0, [&](auto nv) {
            ggx_prefilter_kernel<decltype(nv)::value><<<grid, IBL_THREADS, 0, stream>>>(
                cubemap, atlas, table, cones, atlas + g.levels, atlas + g.weights, p, c0, c0 == 0);
            return launched();
        });
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_ggx_prefilter_adjoint(const float* atlas, const float* level_grad, float* src_grad, float* grad_cubemap,
                                         const TexDims& d, cudaStream_t stream)
{
    IblLevels p = ibl_levels(d);
    if (p.L == 1 || d.TB == 0) return cudaSuccess;
    const GgxLayout g = ggx_layout(d);
    int levels[MIP_MAX_LEVELS], n = 0;
    for (int s = p.ss == 0 ? 0 : 1; s <= p.ss && s < p.L; ++s) levels[n++] = s;
    set_works(p, levels, n);
    const dim3 grid(p.first[p.works], d.TB < IBL_MAX_ITEMS ? d.TB : IBL_MAX_ITEMS);
    for (int c0 = 0; c0 < d.C; c0 += 4) {
        const cudaError_t e = with_nv(d.C - c0, [&](auto nv) {
            ggx_prefilter_adjoint_kernel<decltype(nv)::value><<<grid, IBL_THREADS, 0, stream>>>(
                level_grad, atlas + g.weights, reinterpret_cast<const float4*>(atlas + g.table),
                reinterpret_cast<const float4*>(atlas + g.cones), src_grad, grad_cubemap, p, c0);
            return launched();
        });
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_ggx_brdf_table(float* table, int N, cudaStream_t stream)
{
    ggx_brdf_table_kernel<<<(N * N + 127) / 128, 128, 0, stream>>>(table, N);
    return launched();
}

// the SH projection's scratch: level 0's texel table, then the partial sums
static IblLevels sh_levels(int TB, int S, int C)
{
    IblLevels p = {};
    p.S = S;
    p.TB = TB;
    p.C = C;
    p.L = 1;
    p.table[1] = 6ll * S * S;
    return p;
}

static int cube_sh_chunks(int S) { return (int)((6ll * S * S + CUBE_SH_CHUNK - 1) / CUBE_SH_CHUNK); }

size_t sh_project_scratch_bytes(int TB, int S, int C)
{
    return align_up(sizeof(float4) * 6 * (size_t)S * S, 256) + sizeof(double) * (size_t)TB * cube_sh_chunks(S) * 9 * C;
}

cudaError_t launch_sh_project(const float* cubemap, float* coeffs, void* scratch, int TB, int S, int C, cudaStream_t stream)
{
    const IblLevels p = sh_levels(TB, S, C);
    float4* table = static_cast<float4*>(scratch);
    double* partial = reinterpret_cast<double*>(static_cast<char*>(scratch) + align_up(sizeof(float4) * 6 * (size_t)S * S, 256));
    const int chunks = cube_sh_chunks(S);
    cudaError_t e;
    ggx_texel_table_kernel<<<ibl_blocks(p.table[1]), IBL_THREADS, 0, stream>>>(table, p);
    if ((e = launched()) != cudaSuccess) return e;
    const dim3 grid((unsigned)(chunks < IBL_MAX_BLOCKS ? chunks : IBL_MAX_BLOCKS), TB < IBL_MAX_ITEMS ? TB : IBL_MAX_ITEMS);
    sh_project_partial_kernel<<<grid, IBL_THREADS, 0, stream>>>(cubemap, table, partial, p.table[1], TB, C, chunks);
    if ((e = launched()) != cudaSuccess) return e;
    sh_project_final_kernel<<<ibl_blocks((long long)TB * 9 * C), IBL_THREADS, 0, stream>>>(partial, coeffs, TB, C, chunks);
    return launched();
}

cudaError_t launch_sh_project_backward(const float* grad_coeffs, float* grad_cubemap, void* scratch, int TB, int S, int C,
                                       cudaStream_t stream)
{
    const IblLevels p = sh_levels(TB, S, C);
    float4* table = static_cast<float4*>(scratch);
    cudaError_t e;
    ggx_texel_table_kernel<<<ibl_blocks(p.table[1]), IBL_THREADS, 0, stream>>>(table, p);
    if ((e = launched()) != cudaSuccess) return e;
    sh_project_backward_kernel<<<ibl_blocks((long long)TB * p.table[1] * C), IBL_THREADS, 0, stream>>>(
        table, grad_coeffs, grad_cubemap, p.table[1], TB, C);
    return launched();
}

}  // namespace dirt
