// lighting.cu -- the reflectance models of dirt_b200/lighting.py (dirt_lighting_forward / dirt_lighting_backward):
// Lambert under a directional light, Phong under a directional light, Lambert under a point light, each as one pass over
// the points (DESIGN.md §7.2).
//
// One thread per point; a CTA holds 256 points of one item (blockIdx.x = chunk of the item, blockIdx.y = item, looping
// past the grid limit).  The 12-byte rows (normals, positions, and colours / grad_out / outputs when C = 3) are staged
// through the warp's slice of shared memory, so that each global access of the warp covers consecutive floats.
// Backward recomputes the forward from the inputs.  Gradients of parameters shared by many points (light, light colour,
// camera, shininess) are summed without atomics: each CTA writes its sums to its own row of the partials, then one
// small kernel adds the rows of each item (or of all items, for a shared parameter) in a fixed order.  Two calls on the
// same inputs therefore give bit-identical parameter gradients.
//
// The file also holds the GGX specular reflectance (dirt_ggx_lighting_forward / _backward, DESIGN.md §7.9) and the
// spherical-harmonics environment lighting (dirt_sh_lighting_forward / _backward, DESIGN.md §7.8), which use the same
// staging, per-CTA partials and reduction kernel, and the tangent-space normal mapping (dirt_normal_map_forward /
// _backward, DESIGN.md §7.14), which uses the same staging and grid.
#include "../../include/dirt_b200.h"
#include "common.cuh"

namespace dirt {

namespace {

constexpr int WARPS = LIGHT_THREADS / 32;
constexpr int RED_SLOTS = 4;                 // values per reduction round (light, camera: 3; shininess, one channel: 1)
constexpr unsigned FULL = 0xffffffffu;
constexpr int DD = DIRT_LIGHT_DIFFUSE_DIRECTIONAL, SP = DIRT_LIGHT_SPECULAR_DIRECTIONAL, DP = DIRT_LIGHT_DIFFUSE_POINT;
constexpr int REDUCE_THREADS = 256;
#ifndef DIRT_LIGHT_MAX_ITEMS_PER_GRID
#define DIRT_LIGHT_MAX_ITEMS_PER_GRID 65535
#endif
constexpr unsigned MAX_ITEMS_PER_GRID = DIRT_LIGHT_MAX_ITEMS_PER_GRID;   // gridDim.y
#ifndef DIRT_LIGHT_REDUCE_MAX_BLOCKS
#define DIRT_LIGHT_REDUCE_MAX_BLOCKS (1ll << 20)
#endif
constexpr long long REDUCE_MAX_BLOCKS = DIRT_LIGHT_REDUCE_MAX_BLOCKS;   // lighting_reduce_kernel loops beyond this

// dot product in a fixed order: fma(a2, b2, fma(a1, b1, a0 * b0))
__device__ __forceinline__ float dot3(const float a[3], const float b[3])
{
    return __fmaf_rn(a[2], b[2], __fmaf_rn(a[1], b[1], __fmul_rn(a[0], b[0])));
}

// abs(cos) (double-sided) or clamp(cos, min=0), NaN passing through as in torch
template <bool DS>
__device__ __forceinline__ float cos_term(float c)
{
    return DS ? fabsf(c) : (c < 0.f ? 0.f : c);
}
// torch's derivative of cos_term: sgn (0 at 0 and at NaN) or the mask cos >= 0 (1 at exactly 0, 0 at NaN)
template <bool DS>
__device__ __forceinline__ float cos_term_grad(float c)
{
    return DS ? (c > 0.f ? 1.f : (c < 0.f ? -1.f : 0.f)) : (c >= 0.f ? 1.f : 0.f);
}

// The forward's intermediates of one point.  f multiplies every channel: out_c = (light_color_c * color_c) * f.
struct Shade {
    float L[3];                  // light direction (directional models) or position (point light)
    float cos, t, f;             // cosine, its term, the channel factor (t, or pow(t, s) for Phong)
    float s;                     // Phong: shininess
    float two_dot, r[3];         // Phong: 2 (n . -L), reflected = L + two_dot * n
    float tc[3], norm, u[3];     // Phong: to_camera = camera - p, |to_camera|, to_camera / norm + 1e-12
    float rel[3], nr, d, inc[3]; // point light: p - light, |rel|, |rel| + 1e-12, rel / d
};

__device__ __forceinline__ const float* item_row(const float* p, bool per_item, long long b, int k)
{
    return p + (per_item ? b * k : 0);
}

template <int MODEL, bool DS>
__device__ __forceinline__ Shade shade(const LightArgs& a, long long b, const float n[3], const float p[3])
{
    Shade h;
    const float* L = item_row(a.light, a.item_light, b, 3);
#pragma unroll
    for (int i = 0; i < 3; ++i) h.L[i] = __ldg(L + i);
    if (MODEL == DD) {
        const float m[3] = {-h.L[0], -h.L[1], -h.L[2]};
        h.cos = dot3(n, m);
        h.t = h.f = cos_term<DS>(h.cos);
    } else if (MODEL == SP) {
        const float m[3] = {-h.L[0], -h.L[1], -h.L[2]};
        h.two_dot = __fmul_rn(2.f, dot3(n, m));
        const float* cam = item_row(a.camera, a.item_camera, b, 3);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            h.r[i] = __fadd_rn(h.L[i], __fmul_rn(h.two_dot, n[i]));
            h.tc[i] = __fsub_rn(__ldg(cam + i), p[i]);
        }
        h.norm = __fsqrt_rn(dot3(h.tc, h.tc));
#pragma unroll
        for (int i = 0; i < 3; ++i) h.u[i] = __fadd_rn(__fdiv_rn(h.tc[i], h.norm), 1.e-12f);
        h.cos = dot3(h.u, h.r);
        h.t = cos_term<DS>(h.cos);
        h.s = __ldg(item_row(a.shininess, a.item_shininess, b, 1));
        h.f = powf(h.t, h.s);
    } else {
#pragma unroll
        for (int i = 0; i < 3; ++i) h.rel[i] = __fsub_rn(p[i], h.L[i]);
        h.nr = __fsqrt_rn(dot3(h.rel, h.rel));
        h.d = __fadd_rn(h.nr, 1.e-12f);
#pragma unroll
        for (int i = 0; i < 3; ++i) h.inc[i] = __fdiv_rn(h.rel[i], h.d);
        h.cos = dot3(n, h.inc);
        h.t = h.f = cos_term<DS>(h.cos);
    }
    return h;
}

// ---- forward --------------------------------------------------------------------------------------------------------

// CT = 3 (colours and outputs staged like the other rows) or 0 (any C, one channel at a time)
template <int MODEL, bool DS, int CT>
__global__ void __launch_bounds__(LIGHT_THREADS) lighting_forward_kernel(LightArgs a)
{
    __shared__ float stage[LIGHT_THREADS * 3];
    const int lane = threadIdx.x & 31;
    float* s = stage + (threadIdx.x & ~31) * 3;
    const long long v0 = (long long)blockIdx.x * LIGHT_THREADS + (threadIdx.x & ~31);
    if (v0 >= a.V) return;   // the whole warp
    const int n = (int)(a.V - v0 < 32 ? a.V - v0 : 32);
    const int C = CT ? CT : a.C;
    for (long long b = blockIdx.y; b < a.B; b += gridDim.y) {
        const long long row0 = b * a.V + v0, row = row0 + lane;
        float nrm[3], pos[3] = {0.f, 0.f, 0.f};
        stage_load<3>(a.normals, a.sn, row0, n, s, lane, nrm);
        if (MODEL != DD) stage_load<3>(a.positions, a.sp, row0, n, s, lane, pos);
        const Shade h = shade<MODEL, DS>(a, b, nrm, pos);
        const float* lc = item_row(a.light_color, a.item_color, b, C);
        if (CT == 3) {
            float k[3], o[3];
            stage_load<3>(a.colors, a.sc, row0, n, s, lane, k);
#pragma unroll
            for (int c = 0; c < 3; ++c) o[c] = __fmul_rn(__fmul_rn(__ldg(lc + c), k[c]), h.f);
            stage_store<3>(a.out, row0, n, s, lane, o);
        } else if (lane < n) {
            for (int c = 0; c < C; ++c)
                a.out[row * C + c] = __fmul_rn(__fmul_rn(__ldg(lc + c), __ldg(a.colors + row * a.sc + c)), h.f);
        }
    }
}

// ---- backward -------------------------------------------------------------------------------------------------------

// Sums NV values over the CTA in a fixed order (a butterfly in each warp, then the warps in order) and has thread j write
// the j-th sum to dst[j].  Block-collective.
template <int NV>
__device__ __forceinline__ void cta_partial(const float v[NV], float* red, float* dst)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
        float x = v[j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(FULL, x, o);
        if (lane == 0) red[warp * RED_SLOTS + j] = x;
    }
    __syncthreads();
    if (threadIdx.x < NV) {
        float x = red[threadIdx.x];
#pragma unroll
        for (int w = 1; w < WARPS; ++w) x += red[w * RED_SLOTS + threadIdx.x];
        dst[threadIdx.x] = x;
    }
    __syncthreads();
}

template <int MODEL, bool DS, int CT>
__global__ void __launch_bounds__(LIGHT_THREADS) lighting_backward_kernel(LightArgs a)
{
    __shared__ float stage[LIGHT_THREADS * 3];
    __shared__ float red[WARPS * RED_SLOTS];
    const int lane = threadIdx.x & 31;
    float* s = stage + (threadIdx.x & ~31) * 3;
    const long long v0 = (long long)blockIdx.x * LIGHT_THREADS + (threadIdx.x & ~31);
    const int n = v0 >= a.V ? 0 : (int)(a.V - v0 < 32 ? a.V - v0 : 32);   // warp-uniform; 0: the warp only helps reduce
    const bool live = lane < n;
    const int C = CT ? CT : a.C;
    const int P = LIGHT_FIXED_PARAMS + a.C;
    for (long long b = blockIdx.y; b < a.B; b += gridDim.y) {
        const long long row0 = b * a.V + v0, row = row0 + lane;
        float nrm[3] = {0.f, 0.f, 0.f}, pos[3] = {0.f, 0.f, 0.f};
        if (n) {
            stage_load<3>(a.normals, a.sn, row0, n, s, lane, nrm);
            if (MODEL != DD) stage_load<3>(a.positions, a.sp, row0, n, s, lane, pos);
        }
        const Shade h = shade<MODEL, DS>(a, b, nrm, pos);
        const float* lc = item_row(a.light_color, a.item_color, b, C);

        // out_c = q_c * f with q_c = light_color_c * color_c:  d/df = sum_c g_c q_c, d/dq_c = g_c f
        float gf = 0.f, glc3[3] = {0.f, 0.f, 0.f};
        if (CT == 3) {
            float g[3] = {0.f, 0.f, 0.f}, k[3] = {0.f, 0.f, 0.f}, gk[3];
            if (n) {
                stage_load<3>(a.grad_out, 3, row0, n, s, lane, g);
                stage_load<3>(a.colors, a.sc, row0, n, s, lane, k);
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float l = __ldg(lc + c), gq = g[c] * h.f;
                gf += g[c] * (l * k[c]);
                gk[c] = gq * l;
                glc3[c] = live ? gq * k[c] : 0.f;
            }
            if (a.g_colors && n) stage_store<3>(a.g_colors, row0, n, s, lane, gk);
        } else if (live) {
            for (int c = 0; c < C; ++c) {
                const float l = __ldg(lc + c), g = __ldg(a.grad_out + row * C + c);
                gf += g * (l * __ldg(a.colors + row * a.sc + c));
                if (a.g_colors) a.g_colors[row * C + c] = (g * h.f) * l;
            }
        }

        // the scalar chain down to the cosine, then to the per-point inputs and the parameters
        float gn[3], gp[3] = {0.f, 0.f, 0.f}, gL[3], gcam[3] = {0.f, 0.f, 0.f}, gs = 0.f;
        float gt = gf;
        if (MODEL == SP) {
            // torch's pow backward: no gradient through an exponent of 0, none to the exponent at base 0 (exponent >= 0)
            gt = h.s == 0.f ? 0.f : gf * (h.s * powf(h.t, h.s - 1.f));
            gs = gf * ((h.t == 0.f && h.s >= 0.f) ? 0.f : h.f * logf(h.t));
        }
        const float gc = gt * cos_term_grad<DS>(h.cos);
        if (MODEL == DD) {
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                gn[i] = gc * -h.L[i];
                gL[i] = -(gc * nrm[i]);
            }
        } else if (MODEL == SP) {
            float gu[3], gnorm = 0.f, g2d = 0.f;
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                gu[i] = gc * h.r[i];
                const float gr = gc * h.u[i];
                gL[i] = gr;
                g2d += gr * nrm[i];
                gn[i] = gr * h.two_dot;
                gnorm -= gu[i] * h.tc[i] / (h.norm * h.norm);
            }
            const float gdot = 2.f * g2d;
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                gn[i] += gdot * -h.L[i];
                gL[i] -= gdot * nrm[i];
                // torch's norm backward has no gradient at a zero vector
                const float gtc = gu[i] / h.norm + (h.norm == 0.f ? 0.f : h.tc[i] * (gnorm / h.norm));
                gcam[i] = gtc;
                gp[i] = -gtc;
            }
        } else {
            float gd = 0.f, grel[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                gn[i] = gc * h.inc[i];
                const float ginc = gc * nrm[i];
                grel[i] = ginc / h.d;
                gd -= ginc * h.rel[i] / (h.d * h.d);
            }
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                gp[i] = grel[i] + (h.nr == 0.f ? 0.f : h.rel[i] * (gd / h.nr));
                gL[i] = -gp[i];
            }
        }
        if (n) {
            if (a.g_normals) stage_store<3>(a.g_normals, row0, n, s, lane, gn);
            if (MODEL != DD && a.g_positions) stage_store<3>(a.g_positions, row0, n, s, lane, gp);
        }

        // this CTA's sums of the parameter gradients (lanes without a point add zeros)
        if (a.partial) {
            float* dst = a.partial + ((long long)b * a.chunks + blockIdx.x) * P;
            if (a.g_light) {
                const float v[3] = {live ? gL[0] : 0.f, live ? gL[1] : 0.f, live ? gL[2] : 0.f};
                cta_partial<3>(v, red, dst);
            }
            if (a.g_light_color) {
                if (CT == 3) {
                    cta_partial<3>(glc3, red, dst + 3);
                } else {
                    for (int c = 0; c < C; ++c) {
                        const float v[1] = {live ? (__ldg(a.grad_out + row * C + c) * h.f) *
                                                       __ldg(a.colors + row * a.sc + c) : 0.f};
                        cta_partial<1>(v, red, dst + 3 + c);
                    }
                }
            }
            if (MODEL == SP && a.g_camera) {
                const float v[3] = {live ? gcam[0] : 0.f, live ? gcam[1] : 0.f, live ? gcam[2] : 0.f};
                cta_partial<3>(v, red, dst + 3 + C);
            }
            if (MODEL == SP && a.g_shininess) {
                const float v[1] = {live ? gs : 0.f};
                cta_partial<1>(v, red, dst + 6 + C);
            }
        }
    }
}

// One CTA per element of a wanted parameter gradient: the sum of its column of the partials over the rows of its item
// (per-item parameter) or of every item (shared parameter), each thread taking a fixed stride of rows and the CTA
// adding the threads' sums as a fixed tree.
struct ReduceJobs {
    float* out[4];
    int offset[4];           // column of the partials
    int width[4];
    bool per_item[4];
    long long first[5];      // first output element of each job; first[count] = total
    int count;
};

__global__ void __launch_bounds__(REDUCE_THREADS) lighting_reduce_kernel(const float* __restrict__ partial, ReduceJobs jobs,
                                                                         long long total, long long chunks, int B, int P)
{
    __shared__ float sum[REDUCE_THREADS];
    for (long long e = blockIdx.x; e < total; e += gridDim.x) {
        // the job of element e, selected without indexing the parameter struct dynamically (which needs a stack copy)
        float* out = jobs.out[0];
        long long first = 0;
        int offset = jobs.offset[0], width = jobs.width[0];
        bool per_item = jobs.per_item[0];
#pragma unroll
        for (int j = 1; j < 4; ++j)
            if (j < jobs.count && e >= jobs.first[j]) {
                out = jobs.out[j]; first = jobs.first[j]; offset = jobs.offset[j]; width = jobs.width[j];
                per_item = jobs.per_item[j];
            }
        const long long local = e - first;
        const long long item = per_item ? local / width : 0;
        const int col = offset + (int)(local - item * width);
        const long long r0 = per_item ? item * chunks : 0, rows = per_item ? chunks : B * chunks;
        float x = 0.f;
        for (long long i = threadIdx.x; i < rows; i += REDUCE_THREADS) x += partial[(r0 + i) * P + col];
        sum[threadIdx.x] = x;
        __syncthreads();
#pragma unroll
        for (int h = REDUCE_THREADS / 2; h > 0; h >>= 1) {
            if (threadIdx.x < h) sum[threadIdx.x] += sum[threadIdx.x + h];
            __syncthreads();
        }
        if (threadIdx.x == 0) out[local] = sum[0];
        __syncthreads();
    }
}

template <int MODEL, bool DS>
void forward_md(const LightArgs& a, cudaStream_t stream)
{
    if (a.C == 3) lighting_forward_kernel<MODEL, DS, 3><<<light_grid(a.chunks, a.B), LIGHT_THREADS, 0, stream>>>(a);
    else lighting_forward_kernel<MODEL, DS, 0><<<light_grid(a.chunks, a.B), LIGHT_THREADS, 0, stream>>>(a);
}

template <int MODEL, bool DS>
void backward_md(const LightArgs& a, cudaStream_t stream)
{
    if (a.C == 3) lighting_backward_kernel<MODEL, DS, 3><<<light_grid(a.chunks, a.B), LIGHT_THREADS, 0, stream>>>(a);
    else lighting_backward_kernel<MODEL, DS, 0><<<light_grid(a.chunks, a.B), LIGHT_THREADS, 0, stream>>>(a);
}

template <int MODEL>
void forward_m(const LightArgs& a, cudaStream_t stream)
{
    if (a.double_sided) forward_md<MODEL, true>(a, stream);
    else forward_md<MODEL, false>(a, stream);
}

template <int MODEL>
void backward_m(const LightArgs& a, cudaStream_t stream)
{
    if (a.double_sided) backward_md<MODEL, true>(a, stream);
    else backward_md<MODEL, false>(a, stream);
}

// The reduction jobs of the wanted parameter gradients of a partial row [light (3), light colour (C), camera (3),
// shininess (1)]; camera and shininess only where the model has them.
ReduceJobs param_jobs(const LightArgs& a, bool camera, bool shininess)
{
    ReduceJobs jobs;
    jobs.count = 0;
    jobs.first[0] = 0;
    auto add = [&](float* out, int offset, int width, bool per_item) {
        if (!out) return;
        const int k = jobs.count++;
        jobs.out[k] = out; jobs.offset[k] = offset; jobs.width[k] = width; jobs.per_item[k] = per_item;
        jobs.first[k + 1] = jobs.first[k] + (per_item ? (long long)a.B : 1ll) * width;
    };
    add(a.g_light, 0, 3, a.item_light);
    add(a.g_light_color, 3, a.C, a.item_color);
    if (camera) add(a.g_camera, 3 + a.C, 3, a.item_camera);
    if (shininess) add(a.g_shininess, 6 + a.C, 1, a.item_shininess);
    return jobs;
}

// with no points: zeroes the jobs' outputs
cudaError_t zero_params(const ReduceJobs& jobs, cudaStream_t stream)
{
    cudaError_t e;
    for (int k = 0; k < jobs.count; ++k) {
        const size_t bytes = sizeof(float) * (size_t)(jobs.first[k + 1] - jobs.first[k]);
        if (bytes && (e = cudaMemsetAsync(jobs.out[k], 0, bytes, stream)) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// after the point kernel: adds the partial rows of every job in a fixed order
cudaError_t reduce_params(const LightArgs& a, const ReduceJobs& jobs, cudaStream_t stream)
{
    if (!jobs.count) return cudaSuccess;
    const long long total = jobs.first[jobs.count];
    const unsigned blocks = (unsigned)(total < REDUCE_MAX_BLOCKS ? total : REDUCE_MAX_BLOCKS);
    lighting_reduce_kernel<<<blocks, REDUCE_THREADS, 0, stream>>>(a.partial, jobs, total, a.chunks, a.B,
                                                                  LIGHT_FIXED_PARAMS + a.C);
    return launched();
}

}  // namespace

dim3 light_grid(long long chunks, int B)
{
    return dim3((unsigned)chunks, (unsigned)(B < (int)MAX_ITEMS_PER_GRID ? B : (int)MAX_ITEMS_PER_GRID));
}

cudaError_t launch_partials_reduce(const float* partial, float* out, int width, bool per_item, long long chunks, int B,
                                   cudaStream_t stream)
{
    ReduceJobs jobs = {};
    jobs.count = 1;
    jobs.out[0] = out; jobs.offset[0] = 0; jobs.width[0] = width; jobs.per_item[0] = per_item;
    const long long total = (per_item ? (long long)B : 1ll) * width;
    jobs.first[0] = 0; jobs.first[1] = total;
    const unsigned blocks = (unsigned)(total < REDUCE_MAX_BLOCKS ? total : REDUCE_MAX_BLOCKS);
    lighting_reduce_kernel<<<blocks, REDUCE_THREADS, 0, stream>>>(partial, jobs, total, chunks, B, width);
    return launched();
}

cudaError_t launch_lighting_forward(const LightArgs& a, cudaStream_t stream)
{
    if ((long long)a.B * a.V == 0) return cudaSuccess;
    switch (a.model) {
        case DD: forward_m<DD>(a, stream); break;
        case SP: forward_m<SP>(a, stream); break;
        default: forward_m<DP>(a, stream);
    }
    return launched();
}

cudaError_t launch_lighting_backward(const LightArgs& a, cudaStream_t stream)
{
    const bool sp = a.model == SP;
    const ReduceJobs jobs = param_jobs(a, sp, sp);
    cudaError_t e;
    if ((long long)a.B * a.V == 0) return zero_params(jobs, stream);
    const bool per_point = a.g_normals || a.g_colors || (a.model != DD && a.g_positions);
    if (!per_point && !jobs.count) return cudaSuccess;
    LightArgs b = a;
    if (!jobs.count) b.partial = nullptr;
    switch (a.model) {
        case DD: backward_m<DD>(b, stream); break;
        case SP: backward_m<SP>(b, stream); break;
        default: backward_m<DP>(b, stream);
    }
    if ((e = launched()) != cudaSuccess) return e;
    return reduce_params(b, jobs, stream);
}

// ---- GGX microfacet specular reflectance (dirt_ggx_lighting_*, DESIGN.md §7.9) ---------------------------------------
//
// out_c = pi * light_color_c * F_c * D * Vis * NdotL on lit points (NdotL > 0 and NdotV > 0), else 0: Trowbridge-Reitz D,
// height-correlated Smith Vis, Schlick F.  Laid out as lighting_forward_kernel / lighting_backward_kernel, with the
// roughness read directly (one float per point) and the specular colour F0 in place of the colours.  The geometry of a
// point and the scalar chain down to f = pi D Vis NdotL are evaluated in double precision: near the centre of a sharp
// highlight D changes by a relative 2 / a^2 per radian between n and h (about 1000 at the roughness clamp), so fp32
// rounding of the unit vectors alone (a few 1e-8 rad) would cost about 1e-4 in D and more in its gradient.  The channel
// loop is fp32.  The backward pass recomputes the forward; the parameter gradients go through cta_partial and
// lighting_reduce_kernel as the other models'.

namespace {

constexpr float GGX_MIN_ROUGHNESS = 0.045f;
constexpr double GGX_PI = 3.14159265358979323846;

struct UnitVec {
    double u[3], norm;   // u = x / (|x| + 1e-12), norm = |x|
};

__device__ __forceinline__ double ddot3(const double a[3], const double b[3])
{
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
}

__device__ __forceinline__ UnitVec unit_vec(const double x[3])
{
    UnitVec y;
    y.norm = sqrt(ddot3(x, x));
    const double inv = 1.0 / (y.norm + 1e-12);
#pragma unroll
    for (int i = 0; i < 3; ++i) y.u[i] = x[i] * inv;
    return y;
}

// gx from gu through u = x / (|x| + 1e-12): gu / (|x| + 1e-12) - u (u . gu) / |x|, as torch: no gradient through the
// norm of a zero vector
__device__ __forceinline__ void unit_grad(const UnitVec& y, const double gu[3], double gx[3])
{
    const double inv = 1.0 / (y.norm + 1e-12), t = y.norm == 0.0 ? 0.0 : ddot3(y.u, gu) / y.norm;
#pragma unroll
    for (int i = 0; i < 3; ++i) gx[i] = gu[i] * inv - y.u[i] * t;
}

__device__ __forceinline__ void cross3(const double a[3], const double b[3], double c[3])
{
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

// The forward's intermediates of one point.  The channel factors: out_c = light_color_c (F0_c + (1 - F0_c) m5) f.
struct Ggx {
    UnitVec n, v, l, h;           // n.u: the normal after the double-sided flip s
    double s;
    double NL, NV, NH, VH, cr[3]; // cr = n x h
    double a, a2, A, k, D, GV, GL, den, Vis, m;
    float f, m5;                  // f = pi D Vis NdotL (0 where not lit), m5 = (1 - VdotH)^5
    bool lit;
};

template <bool POINT, bool DS>
__device__ __forceinline__ Ggx ggx_shade(const LightArgs& a, long long b, const float n[3], const float p[3], float r)
{
    Ggx g;
    const float* L = item_row(a.light, a.item_light, b, 3);
    const float* cam = item_row(a.camera, a.item_camera, b, 3);
    double x[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) x[i] = n[i];
    g.n = unit_vec(x);
#pragma unroll
    for (int i = 0; i < 3; ++i) x[i] = (double)__ldg(cam + i) - (double)p[i];
    g.v = unit_vec(x);
#pragma unroll
    for (int i = 0; i < 3; ++i) x[i] = POINT ? (double)__ldg(L + i) - (double)p[i] : -(double)__ldg(L + i);
    g.l = unit_vec(x);
    // turned to face the camera (no flip at exactly 0)
    g.s = DS && ddot3(g.n.u, g.v.u) < 0.0 ? -1.0 : 1.0;
#pragma unroll
    for (int i = 0; i < 3; ++i) g.n.u[i] *= g.s;
    g.NV = ddot3(g.n.u, g.v.u);
    g.NL = ddot3(g.n.u, g.l.u);
    g.lit = g.NL > 0.0 && g.NV > 0.0;
#pragma unroll
    for (int i = 0; i < 3; ++i) x[i] = g.l.u[i] + g.v.u[i];
    g.h = unit_vec(x);
    g.NH = ddot3(g.n.u, g.h.u);
    g.VH = ddot3(g.v.u, g.h.u);
    cross3(g.n.u, g.h.u, g.cr);
    g.a = r < GGX_MIN_ROUGHNESS ? (double)GGX_MIN_ROUGHNESS : (double)r;   // NaN passes through, as torch's clamp
    g.a2 = g.a * g.a;
    g.A = g.a2 * g.a2;
    // k = A NdotH^2 + |n x h|^2 rather than NdotH^2 (A - 1) + 1, which cancels for small A
    g.k = g.A * g.NH * g.NH + ddot3(g.cr, g.cr);
    g.D = g.A / (GGX_PI * g.k * g.k);
    g.GV = sqrt(g.NV * g.NV * (1.0 - g.A) + g.A);
    g.GL = sqrt(g.NL * g.NL * (1.0 - g.A) + g.A);
    g.den = g.NL * g.GV + g.NV * g.GL;
    g.Vis = 0.5 / g.den;
    g.m = 1.0 - g.VH;
    const double m2 = g.m * g.m;
    g.m5 = (float)(m2 * m2 * g.m);
    g.f = g.lit ? (float)(GGX_PI * g.D * g.Vis * g.NL) : 0.f;
    return g;
}

__device__ __forceinline__ float ggx_fresnel(float F0, float m5)
{
    return F0 + (1.f - F0) * m5;
}

// CT = 3 (specular colours and outputs staged like the other rows) or 0 (any C, one channel at a time)
template <bool POINT, bool DS, int CT>
__global__ void __launch_bounds__(LIGHT_THREADS) ggx_forward_kernel(LightArgs a)
{
    __shared__ float stage[LIGHT_THREADS * 3];
    const int lane = threadIdx.x & 31;
    float* s = stage + (threadIdx.x & ~31) * 3;
    const long long v0 = (long long)blockIdx.x * LIGHT_THREADS + (threadIdx.x & ~31);
    if (v0 >= a.V) return;   // the whole warp
    const int n = (int)(a.V - v0 < 32 ? a.V - v0 : 32);
    const int C = CT ? CT : a.C;
    for (long long b = blockIdx.y; b < a.B; b += gridDim.y) {
        const long long row0 = b * a.V + v0, row = row0 + lane;
        float nrm[3], pos[3];
        stage_load<3>(a.normals, a.sn, row0, n, s, lane, nrm);
        stage_load<3>(a.positions, a.sp, row0, n, s, lane, pos);
        const float r = lane < n ? __ldg(a.roughness + row * a.sr) : 0.f;
        const Ggx g = ggx_shade<POINT, DS>(a, b, nrm, pos, r);
        const float* lc = item_row(a.light_color, a.item_color, b, C);
        if (CT == 3) {
            float F0[3], o[3];
            stage_load<3>(a.colors, a.sc, row0, n, s, lane, F0);
#pragma unroll
            for (int c = 0; c < 3; ++c) o[c] = g.lit ? __ldg(lc + c) * ggx_fresnel(F0[c], g.m5) * g.f : 0.f;
            stage_store<3>(a.out, row0, n, s, lane, o);
        } else if (lane < n) {
            for (int c = 0; c < C; ++c)
                a.out[row * C + c] =
                    g.lit ? __ldg(lc + c) * ggx_fresnel(__ldg(a.colors + row * a.sc + c), g.m5) * g.f : 0.f;
        }
    }
}

template <bool POINT, bool DS, int CT>
__global__ void __launch_bounds__(LIGHT_THREADS) ggx_backward_kernel(LightArgs a)
{
    __shared__ float stage[LIGHT_THREADS * 3];
    __shared__ float red[WARPS * RED_SLOTS];
    const int lane = threadIdx.x & 31;
    float* s = stage + (threadIdx.x & ~31) * 3;
    const long long v0 = (long long)blockIdx.x * LIGHT_THREADS + (threadIdx.x & ~31);
    const int n = v0 >= a.V ? 0 : (int)(a.V - v0 < 32 ? a.V - v0 : 32);   // warp-uniform; 0: the warp only helps reduce
    const bool live = lane < n;
    const int C = CT ? CT : a.C;
    const int P = LIGHT_FIXED_PARAMS + a.C;
    for (long long b = blockIdx.y; b < a.B; b += gridDim.y) {
        const long long row0 = b * a.V + v0, row = row0 + lane;
        float nrm[3] = {0.f, 0.f, 0.f}, pos[3] = {0.f, 0.f, 0.f};
        if (n) {
            stage_load<3>(a.normals, a.sn, row0, n, s, lane, nrm);
            stage_load<3>(a.positions, a.sp, row0, n, s, lane, pos);
        }
        const float r = live ? __ldg(a.roughness + row * a.sr) : 0.f;
        const Ggx g = ggx_shade<POINT, DS>(a, b, nrm, pos, r);
        const bool lit = live && g.lit;
        const float* lc = item_row(a.light_color, a.item_color, b, C);

        // out_c = q_c f with q_c = light_color_c F_c, F_c = F0_c + (1 - F0_c) m5:
        // d/df = sum_c g_c q_c, d/dm5 = f sum_c g_c light_color_c (1 - F0_c), d/dF0_c = g_c light_color_c (1 - m5) f
        float gf = 0.f, gm5 = 0.f, glc3[3] = {0.f, 0.f, 0.f};
        if (CT == 3) {
            float go[3] = {0.f, 0.f, 0.f}, F0[3] = {0.f, 0.f, 0.f}, gF0[3];
            if (n) {
                stage_load<3>(a.grad_out, 3, row0, n, s, lane, go);
                stage_load<3>(a.colors, a.sc, row0, n, s, lane, F0);
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float gl = lit ? go[c] * __ldg(lc + c) : 0.f, F = ggx_fresnel(F0[c], g.m5);
                gf += gl * F;
                gm5 += gl * (1.f - F0[c]);
                gF0[c] = lit ? gl * (1.f - g.m5) * g.f : 0.f;
                glc3[c] = lit ? go[c] * F * g.f : 0.f;
            }
            if (a.g_colors && n) stage_store<3>(a.g_colors, row0, n, s, lane, gF0);
        } else if (live) {
            for (int c = 0; c < C; ++c) {
                const float F0 = __ldg(a.colors + row * a.sc + c);
                const float gl = lit ? __ldg(a.grad_out + row * C + c) * __ldg(lc + c) : 0.f;
                gf += gl * ggx_fresnel(F0, g.m5);
                gm5 += gl * (1.f - F0);
                if (a.g_colors) a.g_colors[row * C + c] = lit ? gl * (1.f - g.m5) * g.f : 0.f;
            }
        }

        // the scalar chain down to the unit vectors, then to the per-point inputs and the parameters
        float gn[3] = {0.f, 0.f, 0.f}, gp[3] = {0.f, 0.f, 0.f}, gL[3] = {0.f, 0.f, 0.f}, gcam[3] = {0.f, 0.f, 0.f};
        float gr = 0.f;
        if (lit) {
            const double gfd = gf, gVH = -(double)gm5 * (double)g.f * 5.0 * (g.m * g.m) * (g.m * g.m);
            const double gD = gfd * GGX_PI * g.Vis * g.NL, gVis = gfd * GGX_PI * g.D * g.NL;
            double gNL = gfd * GGX_PI * g.D * g.Vis;
            // Vis = 0.5 / den, den = NL GV + NV GL, G* = sqrt(N*^2 (1 - A) + A)
            const double gden = -gVis * g.Vis / g.den;
            gNL += gden * g.GV;
            double gNV = gden * g.GL;
            const double gQV = gden * g.NL / (2.0 * g.GV), gQL = gden * g.NV / (2.0 * g.GL);
            gNV += gQV * 2.0 * g.NV * (1.0 - g.A);
            gNL += gQL * 2.0 * g.NL * (1.0 - g.A);
            double gA = gQV * (1.0 - g.NV * g.NV) + gQL * (1.0 - g.NL * g.NL);
            // D = A / (pi k^2), k = A NH^2 + |cr|^2
            gA += gD / (GGX_PI * g.k * g.k);
            const double gk = -2.0 * gD * g.D / g.k;
            gA += gk * g.NH * g.NH;
            const double gNH = gk * 2.0 * g.A * g.NH;
            double gcr[3], t[3], gN[3], gh[3], gv[3], gl[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) gcr[i] = 2.0 * gk * g.cr[i];
            cross3(g.h.u, gcr, gN);   // d(n x h)/dn
            cross3(gcr, g.n.u, gh);   // d(n x h)/dh
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                gN[i] += gNH * g.h.u[i] + gNV * g.v.u[i] + gNL * g.l.u[i];
                gh[i] += gNH * g.n.u[i] + gVH * g.v.u[i];
                gv[i] = gVH * g.h.u[i] + gNV * g.n.u[i];
                gl[i] = gNL * g.n.u[i];
            }
            unit_grad(g.h, gh, t);   // h = unit(l + v)
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                gv[i] += t[i];
                gl[i] += t[i];
            }
            unit_grad(g.n, gN, t);   // n = s unit(n_in): the flip's sign twice inside unit_grad, once outside
#pragma unroll
            for (int i = 0; i < 3; ++i) gn[i] = (float)(g.s * t[i]);
            double gtc[3];
            unit_grad(g.v, gv, gtc);   // v = unit(camera - p)
            unit_grad(g.l, gl, t);     // l = unit(light - p) or unit(-light)
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                gcam[i] = (float)gtc[i];
                gp[i] = (float)(POINT ? -gtc[i] - t[i] : -gtc[i]);
                gL[i] = (float)(POINT ? t[i] : -t[i]);
            }
            // A = (a a)^2; torch's clamp passes the gradient at exactly the minimum
            gr = r >= GGX_MIN_ROUGHNESS ? (float)(gA * 4.0 * g.a2 * g.a) : 0.f;
        }
        if (n) {
            if (a.g_normals) stage_store<3>(a.g_normals, row0, n, s, lane, gn);
            if (a.g_positions) stage_store<3>(a.g_positions, row0, n, s, lane, gp);
        }
        if (a.g_roughness && live) a.g_roughness[row] = gr;

        // this CTA's sums of the parameter gradients (lanes without a lit point add zeros)
        if (a.partial) {
            float* dst = a.partial + ((long long)b * a.chunks + blockIdx.x) * P;
            if (a.g_light) cta_partial<3>(gL, red, dst);
            if (a.g_light_color) {
                if (CT == 3) {
                    cta_partial<3>(glc3, red, dst + 3);
                } else {
                    for (int c = 0; c < C; ++c) {
                        const float v[1] = {lit ? __ldg(a.grad_out + row * C + c) *
                                                      ggx_fresnel(__ldg(a.colors + row * a.sc + c), g.m5) * g.f : 0.f};
                        cta_partial<1>(v, red, dst + 3 + c);
                    }
                }
            }
            if (a.g_camera) cta_partial<3>(gcam, red, dst + 3 + C);
        }
    }
}

template <bool POINT, bool DS>
void ggx_launch(const LightArgs& a, bool forward, cudaStream_t stream)
{
    if (forward) {
        if (a.C == 3) ggx_forward_kernel<POINT, DS, 3><<<light_grid(a.chunks, a.B), LIGHT_THREADS, 0, stream>>>(a);
        else ggx_forward_kernel<POINT, DS, 0><<<light_grid(a.chunks, a.B), LIGHT_THREADS, 0, stream>>>(a);
    } else {
        if (a.C == 3) ggx_backward_kernel<POINT, DS, 3><<<light_grid(a.chunks, a.B), LIGHT_THREADS, 0, stream>>>(a);
        else ggx_backward_kernel<POINT, DS, 0><<<light_grid(a.chunks, a.B), LIGHT_THREADS, 0, stream>>>(a);
    }
}

void ggx_dispatch(const LightArgs& a, bool forward, cudaStream_t stream)
{
    if (a.model) {
        if (a.double_sided) ggx_launch<true, true>(a, forward, stream);
        else ggx_launch<true, false>(a, forward, stream);
    } else {
        if (a.double_sided) ggx_launch<false, true>(a, forward, stream);
        else ggx_launch<false, false>(a, forward, stream);
    }
}

}  // namespace

cudaError_t launch_ggx_forward(const LightArgs& a, cudaStream_t stream)
{
    if ((long long)a.B * a.V == 0) return cudaSuccess;
    ggx_dispatch(a, true, stream);
    return launched();
}

cudaError_t launch_ggx_backward(const LightArgs& a, cudaStream_t stream)
{
    const ReduceJobs jobs = param_jobs(a, true, false);
    if ((long long)a.B * a.V == 0) return zero_params(jobs, stream);
    if (!a.g_normals && !a.g_positions && !a.g_colors && !a.g_roughness && !jobs.count) return cudaSuccess;
    LightArgs b = a;
    if (!jobs.count) b.partial = nullptr;
    ggx_dispatch(b, false, stream);
    const cudaError_t e = launched();
    if (e != cudaSuccess) return e;
    return reduce_params(b, jobs, stream);
}

// ---- spherical-harmonics environment lighting (dirt_sh_lighting_*, DESIGN.md §7.8) ------------------------------------
//
// out_c = albedo_c * E_c, E_c = sum_k (w_l(k) * L_kc) * Y_k(n): the real order-2 SH basis (no Condon-Shortley phase) of
// the normal as given, band weights 1, 2/3, 1/4 (the clamped cosine's A_l / pi).  The forward pass is laid out as
// lighting_forward_kernel.  In the backward pass each thread takes SH_POINTS_PER_THREAD points of its item, 256 apart,
// and (C = 3) keeps its sums of the 27 coefficient gradients in registers until one CTA reduction, so the butterflies
// are paid once per SH_CHUNK points instead of once per 256.  The partials are reduced by lighting_reduce_kernel.

namespace {

constexpr float SH_K0 = 0.28209479177387814f, SH_K1 = 0.4886025119029199f, SH_K2 = 1.0925484305920792f,
                SH_K3 = 0.31539156525252005f, SH_K4 = 0.5462742152960396f;

__device__ __forceinline__ float sh_band_weight(int k) { return k == 0 ? 1.f : (k < 4 ? 2.f / 3.f : 0.25f); }

// Y_k(n), k = l^2 + l + m, each product in the restatement's order
__device__ __forceinline__ void sh_basis(const float n[3], float Y[9])
{
    const float x = n[0], y = n[1], z = n[2];
    Y[0] = SH_K0;
    Y[1] = __fmul_rn(SH_K1, y);
    Y[2] = __fmul_rn(SH_K1, z);
    Y[3] = __fmul_rn(SH_K1, x);
    Y[4] = __fmul_rn(__fmul_rn(SH_K2, x), y);
    Y[5] = __fmul_rn(__fmul_rn(SH_K2, y), z);
    Y[6] = __fmul_rn(SH_K3, __fsub_rn(__fmul_rn(__fmul_rn(3.f, z), z), 1.f));
    Y[7] = __fmul_rn(__fmul_rn(SH_K2, x), z);
    Y[8] = __fmul_rn(SH_K4, __fsub_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
}

// E_c = sum_k (w_k L_kc) Y_k in the fixed order k = 0 .. 8; L: the item's [9, C] coefficients (read-only path)
__device__ __forceinline__ float sh_irradiance(const float* __restrict__ L, int C, int c, const float Y[9])
{
    float e = __fmul_rn(__ldg(L + c), Y[0]);
#pragma unroll
    for (int k = 1; k < 9; ++k) e = __fmaf_rn(__fmul_rn(sh_band_weight(k), __ldg(L + k * C + c)), Y[k], e);
    return e;
}

// d/dn of sum_k s_k Y_k(n)  (s_0 has no derivative)
__device__ __forceinline__ void sh_normal_grad(const float n[3], const float s[9], float g[3])
{
    const float x = n[0], y = n[1], z = n[2];
    g[0] = SH_K1 * s[3] + SH_K2 * (y * s[4] + z * s[7]) + (2.f * SH_K4) * (x * s[8]);
    g[1] = SH_K1 * s[1] + SH_K2 * (x * s[4] + z * s[5]) - (2.f * SH_K4) * (y * s[8]);
    g[2] = SH_K1 * s[2] + SH_K2 * (y * s[5] + x * s[7]) + (6.f * SH_K3) * (z * s[6]);
}

__device__ __forceinline__ const float* sh_item(const ShArgs& a, long long b, int C)
{
    return a.coefficients + (a.item_coef ? b * 9 * C : 0);
}

// CT = 3 (albedo and outputs staged like the normals) or 0 (any C, one channel at a time)
template <int CT>
__global__ void __launch_bounds__(LIGHT_THREADS) sh_forward_kernel(ShArgs a)
{
    __shared__ float stage[LIGHT_THREADS * 3];
    const int lane = threadIdx.x & 31;
    float* s = stage + (threadIdx.x & ~31) * 3;
    const long long v0 = (long long)blockIdx.x * LIGHT_THREADS + (threadIdx.x & ~31);
    if (v0 >= a.V) return;   // the whole warp
    const int n = (int)(a.V - v0 < 32 ? a.V - v0 : 32);
    const int C = CT ? CT : a.C;
    for (long long b = blockIdx.y; b < a.B; b += gridDim.y) {
        const long long row0 = b * a.V + v0, row = row0 + lane;
        const float* L = sh_item(a, b, C);
        float nrm[3], Y[9];
        stage_load<3>(a.normals, a.sn, row0, n, s, lane, nrm);
        sh_basis(nrm, Y);
        if (CT == 3) {
            float k[3], o[3];
            stage_load<3>(a.albedo, a.sa, row0, n, s, lane, k);
#pragma unroll
            for (int c = 0; c < 3; ++c) o[c] = __fmul_rn(k[c], sh_irradiance(L, 3, c, Y));
            stage_store<3>(a.out, row0, n, s, lane, o);
        } else if (lane < n) {
            for (int c = 0; c < C; ++c)
                a.out[row * C + c] = __fmul_rn(__ldg(a.albedo + row * a.sa + c), sh_irradiance(L, C, c, Y));
        }
    }
}

// grad_albedo_c = g_c E_c;  grad_n = sum_c g_c albedo_c dE_c/dn;  grad_L_kc = sum over points of g_c albedo_c w_k Y_k,
// each CTA's sum to its own row of the partials (lanes without a point add zeros)
template <int CT>
__global__ void __launch_bounds__(LIGHT_THREADS) sh_backward_kernel(ShArgs a)
{
    __shared__ float stage[LIGHT_THREADS * 3];
    __shared__ float red[WARPS * RED_SLOTS];
    constexpr int NACC = CT == 3 ? 27 : 1;
    const int lane = threadIdx.x & 31;
    float* s = stage + (threadIdx.x & ~31) * 3;
    const int C = CT ? CT : a.C;
    const long long first = (long long)blockIdx.x * SH_CHUNK + (threadIdx.x & ~31);   // the warp's first point
    for (long long b = blockIdx.y; b < a.B; b += gridDim.y) {
        const float* L = sh_item(a, b, C);
        float acc[NACC];
#pragma unroll
        for (int j = 0; j < NACC; ++j) acc[j] = 0.f;
        for (int p = 0; p < SH_POINTS_PER_THREAD; ++p) {
            const long long v0 = first + (long long)p * LIGHT_THREADS;
            if (v0 >= a.V) break;   // warp-uniform
            const int n = (int)(a.V - v0 < 32 ? a.V - v0 : 32);
            const bool live = lane < n;
            const long long row0 = b * a.V + v0, row = row0 + lane;
            float nrm[3], Y[9], sk[9];
            stage_load<3>(a.normals, a.sn, row0, n, s, lane, nrm);
            if (!live) nrm[0] = nrm[1] = nrm[2] = 0.f;
            sh_basis(nrm, Y);
#pragma unroll
            for (int k = 0; k < 9; ++k) sk[k] = 0.f;
            if (CT == 3) {
                float g[3], k3[3], ga[3];
                stage_load<3>(a.grad_out, 3, row0, n, s, lane, g);
                stage_load<3>(a.albedo, a.sa, row0, n, s, lane, k3);
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float h = live ? g[c] * k3[c] : 0.f;
                    if (a.g_albedo) ga[c] = g[c] * sh_irradiance(L, 3, c, Y);
#pragma unroll
                    for (int k = 0; k < 9; ++k) {
                        const float w = sh_band_weight(k);
                        sk[k] += h * (w * __ldg(L + k * 3 + c));
                        acc[k * 3 + c] += h * (w * Y[k]);
                    }
                }
                if (a.g_albedo) stage_store<3>(a.g_albedo, row0, n, s, lane, ga);
            } else if (live) {
                for (int c = 0; c < C; ++c) {
                    const float g = __ldg(a.grad_out + row * C + c), h = g * __ldg(a.albedo + row * a.sa + c);
                    if (a.g_albedo) a.g_albedo[row * C + c] = g * sh_irradiance(L, C, c, Y);
#pragma unroll
                    for (int k = 1; k < 9; ++k) sk[k] += h * (sh_band_weight(k) * __ldg(L + k * C + c));
                }
            }
            if (a.g_normals) {
                float gn[3];
                sh_normal_grad(nrm, sk, gn);
                stage_store<3>(a.g_normals, row0, n, s, lane, gn);
            }
        }
        if (a.partial) {
            float* dst = a.partial + ((long long)b * a.chunks + blockIdx.x) * (9 * C);
            if (CT == 3) {
#pragma unroll
                for (int r = 0; r < 6; ++r) cta_partial<4>(acc + 4 * r, red, dst + 4 * r);
                cta_partial<3>(acc + 24, red, dst + 24);
            } else {
                // one channel at a time: the thread's points again (their rows are still in cache), then 9 reductions
                for (int c = 0; c < C; ++c) {
                    float a9[9];
#pragma unroll
                    for (int k = 0; k < 9; ++k) a9[k] = 0.f;
                    for (int p = 0; p < SH_POINTS_PER_THREAD; ++p) {
                        const long long v = first + (long long)p * LIGHT_THREADS + lane;
                        if (v >= a.V) break;
                        const long long row = b * a.V + v;
                        const float* np = a.normals + row * a.sn;
                        const float nrm[3] = {__ldg(np), __ldg(np + 1), __ldg(np + 2)};
                        float Y[9];
                        sh_basis(nrm, Y);
                        const float h = __ldg(a.grad_out + row * C + c) * __ldg(a.albedo + row * a.sa + c);
#pragma unroll
                        for (int k = 0; k < 9; ++k) a9[k] += h * (sh_band_weight(k) * Y[k]);
                    }
#pragma unroll
                    for (int k = 0; k < 9; ++k) cta_partial<1>(a9 + k, red, dst + k * C + c);
                }
            }
        }
    }
}

}  // namespace

cudaError_t launch_sh_lighting_forward(const ShArgs& a, cudaStream_t stream)
{
    if ((long long)a.B * a.V == 0) return cudaSuccess;
    const dim3 grid = light_grid(light_chunks(a.V), a.B);
    if (a.C == 3) sh_forward_kernel<3><<<grid, LIGHT_THREADS, 0, stream>>>(a);
    else sh_forward_kernel<0><<<grid, LIGHT_THREADS, 0, stream>>>(a);
    return launched();
}

cudaError_t launch_sh_lighting_backward(const ShArgs& a, cudaStream_t stream)
{
    const long long width = 9ll * a.C, total = (a.item_coef ? (long long)a.B : 1ll) * width;
    cudaError_t e;
    if ((long long)a.B * a.V == 0) {
        if (a.g_coef && total && (e = cudaMemsetAsync(a.g_coef, 0, sizeof(float) * (size_t)total, stream)) != cudaSuccess)
            return e;
        return cudaSuccess;
    }
    if (!a.g_normals && !a.g_albedo && !a.g_coef) return cudaSuccess;
    ShArgs b = a;
    if (!a.g_coef) b.partial = nullptr;
    const dim3 grid = light_grid(a.chunks, a.B);
    if (a.C == 3) sh_backward_kernel<3><<<grid, LIGHT_THREADS, 0, stream>>>(b);
    else sh_backward_kernel<0><<<grid, LIGHT_THREADS, 0, stream>>>(b);
    if ((e = launched()) != cudaSuccess) return e;
    if (a.g_coef) {
        // one job: the [9, C] columns of the partials, per item or over every item
        return launch_partials_reduce(b.partial, a.g_coef, (int)width, a.item_coef, a.chunks, a.B, stream);
    }
    return cudaSuccess;
}

// ---- tangent-space normal mapping (dirt_normal_map_*, DESIGN.md §7.14) -----------------------------------------------
//
// n = unit(normal), T = unit(t - (n . t) n) for the tangent's xyz t, s = -1 if its w < 0 else +1,
// out = unit(m.x T + m.y s (n x T) + m.z n) for the tangent-space sample m; unit(x) = x / (|x| + 1e-12).  One thread per
// point, laid out as lighting_forward_kernel; the backward kernel recomputes the forward.  No parameter is shared by
// the points, so there is no reduction.

namespace {

__device__ __forceinline__ void nm_cross(const float a[3], const float b[3], float c[3])
{
    c[0] = __fsub_rn(__fmul_rn(a[1], b[2]), __fmul_rn(a[2], b[1]));
    c[1] = __fsub_rn(__fmul_rn(a[2], b[0]), __fmul_rn(a[0], b[2]));
    c[2] = __fsub_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0]));
}

// u = x / (|x| + 1e-12); returns |x|
__device__ __forceinline__ float nm_unit(const float x[3], float u[3])
{
    const float nr = __fsqrt_rn(dot3(x, x)), d = __fadd_rn(nr, 1.e-12f);
#pragma unroll
    for (int i = 0; i < 3; ++i) u[i] = __fdiv_rn(x[i], d);
    return nr;
}

// torch autograd's gradient of x / (|x| + 1e-12) for the output gradient g (none through the norm of a zero vector)
__device__ __forceinline__ void nm_unit_grad(const float x[3], const float g[3], float gx[3])
{
    const float nr = __fsqrt_rn(dot3(x, x)), d = __fadd_rn(nr, 1.e-12f);
    const float gd = -__fdiv_rn(dot3(g, x), __fmul_rn(d, d));
    const float k = nr == 0.f ? 0.f : __fdiv_rn(gd, nr);
#pragma unroll
    for (int i = 0; i < 3; ++i) gx[i] = __fmaf_rn(x[i], k, __fdiv_rn(g[i], d));
}

// The forward's intermediates of one point.
struct Perturb {
    float n[3], d, x[3], T[3], s, c[3], y[3];   // n, d = n . t, x = t - d n, T, s, c = n x T, y = the sum out normalises
};

__device__ __forceinline__ Perturb perturb(const float nrm[3], const float t[4], const float m[3])
{
    Perturb p;
    nm_unit(nrm, p.n);
    p.d = dot3(p.n, t);
#pragma unroll
    for (int i = 0; i < 3; ++i) p.x[i] = __fsub_rn(t[i], __fmul_rn(p.d, p.n[i]));
    nm_unit(p.x, p.T);
    p.s = t[3] < 0.f ? -1.f : 1.f;
    nm_cross(p.n, p.T, p.c);
#pragma unroll
    for (int i = 0; i < 3; ++i)
        p.y[i] = __fmaf_rn(m[2], p.n[i], __fmaf_rn(__fmul_rn(m[1], p.s), p.c[i], __fmul_rn(m[0], p.T[i])));
    return p;
}

__global__ void __launch_bounds__(LIGHT_THREADS) normal_map_forward_kernel(NormalMapArgs a)
{
    __shared__ float stage[LIGHT_THREADS * 4];
    const int lane = threadIdx.x & 31;
    float* s = stage + (threadIdx.x & ~31) * 4;
    const long long v0 = (long long)blockIdx.x * LIGHT_THREADS + (threadIdx.x & ~31);
    if (v0 >= a.V) return;   // the whole warp
    const int n = (int)(a.V - v0 < 32 ? a.V - v0 : 32);
    for (long long b = blockIdx.y; b < a.B; b += gridDim.y) {
        const long long row0 = b * a.V + v0;
        float nrm[3], t[4], m[3], o[3];
        stage_load<3>(a.normals, a.sn, row0, n, s, lane, nrm);
        stage_load<4>(a.tangents, a.st, row0, n, s, lane, t);
        stage_load<3>(a.samples, a.sm, row0, n, s, lane, m);
        const Perturb p = perturb(nrm, t, m);
        nm_unit(p.y, o);
        stage_store<3>(a.out, row0, n, s, lane, o);
    }
}

__global__ void __launch_bounds__(LIGHT_THREADS) normal_map_backward_kernel(NormalMapArgs a)
{
    __shared__ float stage[LIGHT_THREADS * 4];
    const int lane = threadIdx.x & 31;
    float* s = stage + (threadIdx.x & ~31) * 4;
    const long long v0 = (long long)blockIdx.x * LIGHT_THREADS + (threadIdx.x & ~31);
    if (v0 >= a.V) return;   // the whole warp
    const int n = (int)(a.V - v0 < 32 ? a.V - v0 : 32);
    for (long long b = blockIdx.y; b < a.B; b += gridDim.y) {
        const long long row0 = b * a.V + v0;
        float nrm[3], t[4], m[3], g[3], gy[3];
        stage_load<3>(a.normals, a.sn, row0, n, s, lane, nrm);
        stage_load<4>(a.tangents, a.st, row0, n, s, lane, t);
        stage_load<3>(a.samples, a.sm, row0, n, s, lane, m);
        stage_load<3>(a.grad_out, 3, row0, n, s, lane, g);
        const Perturb p = perturb(nrm, t, m);
        nm_unit_grad(p.y, g, gy);
        if (a.g_samples) {
            float gm[3];
            gm[0] = dot3(gy, p.T);
            gm[1] = __fmul_rn(p.s, dot3(gy, p.c));
            gm[2] = dot3(gy, p.n);
            stage_store<3>(a.g_samples, row0, n, s, lane, gm);
        }
        if (!a.g_normals && !a.g_tangents) continue;
        // y = m.x T + m.y s (n x T) + m.z n: with q = m.y s gy, a . (n x T) gives T x q to n and q x n to T
        float q[3], gT[3], gn[3], tq[3], qn[3], gx[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) q[i] = __fmul_rn(__fmul_rn(m[1], p.s), gy[i]);
        nm_cross(p.T, q, tq);
        nm_cross(q, p.n, qn);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            gT[i] = __fmaf_rn(m[0], gy[i], qn[i]);
            gn[i] = __fmaf_rn(m[2], gy[i], tq[i]);
        }
        nm_unit_grad(p.x, gT, gx);
        // x = t - d n, d = n . t:  g_t = gx - (gx . n) n,  g_n += -d gx - (gx . n) t
        const float gxn = dot3(gx, p.n);
        float gt[4];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            gt[i] = __fsub_rn(gx[i], __fmul_rn(gxn, p.n[i]));
            gn[i] = __fsub_rn(__fsub_rn(gn[i], __fmul_rn(p.d, gx[i])), __fmul_rn(gxn, t[i]));
        }
        gt[3] = 0.f;
        if (a.g_tangents) stage_store<4>(a.g_tangents, row0, n, s, lane, gt);
        if (a.g_normals) {
            float gnrm[3];
            nm_unit_grad(nrm, gn, gnrm);
            stage_store<3>(a.g_normals, row0, n, s, lane, gnrm);
        }
    }
}

}  // namespace

cudaError_t launch_normal_map_forward(const NormalMapArgs& a, cudaStream_t stream)
{
    if ((long long)a.B * a.V == 0) return cudaSuccess;
    normal_map_forward_kernel<<<light_grid(light_chunks(a.V), a.B), LIGHT_THREADS, 0, stream>>>(a);
    return launched();
}

cudaError_t launch_normal_map_backward(const NormalMapArgs& a, cudaStream_t stream)
{
    if ((long long)a.B * a.V == 0 || (!a.g_normals && !a.g_tangents && !a.g_samples)) return cudaSuccess;
    normal_map_backward_kernel<<<light_grid(light_chunks(a.V), a.B), LIGHT_THREADS, 0, stream>>>(a);
    return launched();
}

}  // namespace dirt
