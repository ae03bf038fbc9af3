// texture.cu -- differentiable texture lookup (dirt_texture_sample / dirt_texture_sample_backward): the bilinear and
// nearest lookups of the reference's textured sample, restated in torch by examples/textured.py:sample_texture, whose
// values the forward kernel reproduces bit for bit (DESIGN.md §7.1), and the mipmapped (trilinear) lookup of §7.6.
//
// Forward: one thread per lookup (texture_forward_kernel; bilinear and nearest with any C other than 1..4: one per output
// element).  The index pair arrives as one 8-byte load, the texels through the read-only path, and the output leaves in
// vector stores: float2 / float4 for C = 2 / 4, and for C = 3 the warp's 32 x 3 values are staged in shared memory and
// written as 24 float4.
// Backward: one thread per lookup (texture_backward_kernel).  grad_indices comes from the same texels.  grad_texture is
// aggregated inside the warp before it touches global memory: lanes that hit the same texel (MATCH.ANY on its linear
// index) sum their contributions and the lowest of them issues one reduction (a vector RED for C = 2 / 4).
// Both kernels take MIP as a template parameter: false reads level 0 alone (bilinear or nearest), true the two mip levels
// around the lookup's level of detail.
// Deterministic backward (dirt_texture_sample_backward_deterministic): a radix sort of the lookups by base texel, then
// fixed-order float64 sums per texel; see the section below and DESIGN.md §7.5.
#include "../../include/dirt_b200.h"
#include "common.cuh"
#include "sort.cuh"

#include <type_traits>

namespace dirt {

namespace {

constexpr int TEX_THREADS = 256;
#ifndef DIRT_TEX_MAX_BLOCKS
#define DIRT_TEX_MAX_BLOCKS (1 << 16)
#endif
constexpr long long TEX_MAX_BLOCKS = DIRT_TEX_MAX_BLOCKS;   // grid-stride loops beyond this
constexpr unsigned FULL = 0xffffffffu;

// x mod m with the sign of m (Python / torch.remainder) of an integer-valued x; exact for every int64
__device__ __forceinline__ int wrap(long long x, int m)
{
    if (x >= -2147483647ll - 1 && x <= 2147483647ll) {
        const int r = (int)x % m;
        return r < 0 ? r + m : r;
    }
    const long long r = x % m;
    return (int)(r < 0 ? r + m : r);
}

// The texels and weights of one lookup.  A lookup with a non-finite index is invalid: it reads nothing, returns 0 and
// contributes no gradient; its texel coordinates are 0 so that no address formed from them leaves the texture.
struct Taps {
    long long base;        // first texel of the lookup's texture
    int r0, r1, c0, c1;
    float fr, fc;          // fractions; 0 for nearest
    bool valid;
};

__device__ __forceinline__ Taps taps_of(float ir, float ic, const TexDims& d, long long g)
{
    Taps t;
    t.base = d.TB == 1 ? 0ll : (g / d.N) * d.texels;
    t.r0 = t.r1 = t.c0 = t.c1 = 0;
    t.fr = t.fc = 0.f;
    t.valid = isfinite(ir) && isfinite(ic);
    if (!t.valid) return t;
    if (d.mode == DIRT_TEXTURE_NEAREST) {
        // .long() truncates toward zero (saturating here), then clamp to the texture
        const long long r = __float2ll_rz(ir), c = __float2ll_rz(ic);
        t.r0 = t.r1 = (int)(r < 0 ? 0 : (r > d.TH - 1 ? d.TH - 1 : r));
        t.c0 = t.c1 = (int)(c < 0 ? 0 : (c > d.TW - 1 ? d.TW - 1 : c));
        return t;
    }
    const float flr = floorf(ir), flc = floorf(ic);
    t.fr = __fsub_rn(ir, flr);
    t.fc = __fsub_rn(ic, flc);
    t.r0 = wrap(__float2ll_rz(flr), d.TH);
    t.c0 = wrap(__float2ll_rz(flc), d.TW);
    t.r1 = t.r0 + 1 == d.TH ? 0 : t.r0 + 1;
    t.c1 = t.c0 + 1 == d.TW ? 0 : t.c0 + 1;
    return t;
}

template <bool VEC>
__device__ __forceinline__ float2 load_index(const float* indices, long long g)
{
    if (VEC) return __ldg(reinterpret_cast<const float2*>(indices) + g);
    return make_float2(__ldg(indices + 2 * g), __ldg(indices + 2 * g + 1));
}

// ---- levels of a lookup ---------------------------------------------------------------------------------------------
//
// A bilinear or nearest lookup reads level 0, the texture.  A mipmapped (trilinear) lookup (DESIGN.md §7.6) reads a
// pyramid: level k of L is [TB, TH >> k, TW >> k, C]; levels 1 .. L-1 live in the caller's pyramid buffer (mip_offset).
// Per lookup: lambda from the screen-space derivatives, l = floor(lambda), f = lambda - l, and
// out = (1-f) * bilinear_l + f * bilinear_{l+1}, with level l+1 not read when f == 0.  Level k >= 1 is read at
// (index + 0.5) * 2^-k - 0.5, level 0 at the index itself, so that f == 0 at l == 0 is mode bilinear bit for bit.

// level k's dims: the level-0 dims with TH, TW and texels scaled down
__device__ __forceinline__ TexDims level_dims(const TexDims& d, int k)
{
    TexDims e = d;
    e.TH = d.TH >> k;
    e.TW = d.TW >> k;
    e.texels = d.texels >> (2 * k);
    return e;
}

// level k of the texture (k = 0) or of the pyramid
template <typename T>
__host__ __device__ __forceinline__ T* level_base(T* level0, T* pyramid, const TexDims& d, int k)
{
    return k == 0 ? level0 : pyramid + mip_offset(d, k) * d.C;
}

// (index + 0.5) * 2^-k - 0.5, each operation rounded in that order; the index itself at level 0
__device__ __forceinline__ float level_index(float i, int k)
{
    if (k == 0) return i;
    return __fsub_rn(__fmul_rn(__fadd_rn(i, 0.5f), __int_as_float((127 - k) << 23)), 0.5f);
}

struct Lod {
    int l;      // the finer level read
    float f;    // the weight of level l + 1; 0: level l alone
};

// rho^2 = max(d0^2 + d1^2, d2^2 + d3^2) (NaN if either is), lambda = 0.5 log2(rho^2), NaN -> 0, clamped to [0, L-1]
__device__ __forceinline__ Lod lod_of(float4 v, int L)
{
    const float s0 = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
    const float s1 = __fadd_rn(__fmul_rn(v.z, v.z), __fmul_rn(v.w, v.w));
    const float rho2 = isnan(s0) || isnan(s1) ? __int_as_float(0x7fc00000) : fmaxf(s0, s1);
    float lam = __fmul_rn(0.5f, log2f(rho2));
    lam = isnan(lam) ? 0.f : fminf(fmaxf(lam, 0.f), (float)(L - 1));
    Lod o;
    o.l = (int)floorf(lam);
    o.f = __fsub_rn(lam, (float)o.l);
    return o;
}

template <bool VEC>
__device__ __forceinline__ float4 load_derivatives(const float* derivatives, long long g)
{
    if (VEC) return __ldg(reinterpret_cast<const float4*>(derivatives) + g);
    const float* p = derivatives + 4 * g;
    return make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3));
}

// One lookup's levels: taps and pointers of level l (0) and, for a mipmapped lookup, l + 1 (1; unused when f == 0).
// A bilinear or nearest lookup has level 0 alone, l = 0 and f = 0.
struct Lookup {
    Taps t0, t1;
    const float *p0, *p1;   // the lookup's texture at level l / l + 1
    int w0, w1;             // their widths
    Lod lod;
};

__device__ __forceinline__ Lookup trilinear_of(float2 ix, float4 dv, const float* texture, const float* pyramid,
                                               const TexDims& d, int L, long long g)
{
    Lookup q;
    q.lod = lod_of(dv, L);
    const int l = q.lod.l, l1 = l + 1 < L ? l + 1 : l;
    const TexDims d0 = level_dims(d, l), d1 = level_dims(d, l1);
    q.t0 = taps_of(level_index(ix.x, l), level_index(ix.y, l), d0, g);
    q.t1 = taps_of(level_index(ix.x, l1), level_index(ix.y, l1), d1, g);
    // a finite index can map to a non-finite one only past 3.4e38; such a lookup reads nothing, as a non-finite one
    q.t0.valid = q.t0.valid && q.t1.valid;
    q.p0 = level_base(texture, pyramid, d, l) + q.t0.base * d.C;
    q.p1 = level_base(texture, pyramid, d, l1) + q.t1.base * d.C;
    q.w0 = d0.TW;
    q.w1 = d1.TW;
    return q;
}

// lookup g of a texture with C channels (MIP: its pyramid, derivatives and L levels)
template <bool MIP, bool VEC>
__device__ __forceinline__ Lookup lookup_of(const float* texture, const float* pyramid, const float* indices,
                                            const float* derivatives, const TexDims& d, int C, int L, long long g)
{
    const float2 ix = load_index<VEC>(indices, g);
    if (MIP) return trilinear_of(ix, load_derivatives<VEC>(derivatives, g), texture, pyramid, d, L, g);
    Lookup q;
    q.t0 = taps_of(ix.x, ix.y, d, g);
    q.p0 = texture + q.t0.base * C;
    q.w0 = d.TW;
    q.lod.l = 0;
    q.lod.f = 0.f;
    return q;
}

// ---- forward --------------------------------------------------------------------------------------------------------

// channels c0 .. c0 + NV - 1 of the lookup at taps t of a texture of width TW and C channels: the bilinear blend of the
// four texels, or for nearest the texel (r0, c0) alone
template <int NV, bool VEC>
__device__ __forceinline__ void level_rows(const float* tex, const Taps& t, int TW, int C, int c0, bool nearest, float v[NV])
{
    float t00[NV], t01[NV], t10[NV], t11[NV];
    load_row<NV, VEC>(tex + ((long long)t.r0 * TW + t.c0) * C + c0, t00);
    if (nearest) {
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] = t00[j];
        return;
    }
    load_row<NV, VEC>(tex + ((long long)t.r0 * TW + t.c1) * C + c0, t01);
    load_row<NV, VEC>(tex + ((long long)t.r1 * TW + t.c0) * C + c0, t10);
    load_row<NV, VEC>(tex + ((long long)t.r1 * TW + t.c1) * C + c0, t11);
#pragma unroll
    for (int j = 0; j < NV; ++j) v[j] = bilinear(t00[j], t01[j], t10[j], t11[j], t.fr, t.fc);
}

// Channels c0 .. c0 + NV - 1 of lookup g = base + lane go to out.  Every lane of the warp calls it: for C = 3 the warp's
// values are staged in stage.
template <int CT, bool VEC>
__device__ __forceinline__ void store_out(float* out, float* stage, long long base, int c0, int C, long long total,
                                          const float v[])
{
    constexpr int NV = CT ? CT : 1;
    const int lane = threadIdx.x & 31;
    const long long g = base + lane;
    float* o = out + g * C + c0;
    if (VEC && CT == 4) {
        if (g < total) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1 % NV], v[2 % NV], v[3 % NV]);
    } else if (VEC && CT == 2) {
        if (g < total) *reinterpret_cast<float2*>(o) = make_float2(v[0], v[1 % NV]);
    } else if (VEC && CT == 3 && base + 32 <= total) {
        // the warp's 96 consecutive floats start on a 384-byte boundary: 24 float4 stores
        float* s = stage + (threadIdx.x & ~31) * 3;
#pragma unroll
        for (int j = 0; j < NV; ++j) s[lane * 3 + j] = v[j];
        __syncwarp();
        if (lane < 24) *reinterpret_cast<float4*>(out + base * 3 + lane * 4) = reinterpret_cast<const float4*>(s)[lane];
        __syncwarp();
    } else if (g < total) {
#pragma unroll
        for (int j = 0; j < NV; ++j) o[j] = v[j];
    }
}

// One thread per lookup, CT = C in 1..4, or 0 for any C (MIP only: channels in a loop, scalar accesses).  VEC: the
// pointers are aligned for the vector loads and stores (see forward_ct).  The loop runs per warp, so that the C = 3
// staging sees all 32 lanes.  MIP: pyramid, derivatives and L as in trilinear_of; unused otherwise.
template <int CT, bool VEC, bool MIP>
__global__ void __launch_bounds__(TEX_THREADS) texture_forward_kernel(const float* __restrict__ texture,
                                                                      const float* __restrict__ indices,
                                                                      float* __restrict__ out, TexDims d,
                                                                      const float* __restrict__ pyramid,
                                                                      const float* __restrict__ derivatives, int L)
{
    constexpr int NV = CT ? CT : 1;
    const int C = CT ? CT : d.C;
    __shared__ __align__(16) float stage[CT == 3 ? TEX_THREADS * 3 : 1];
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long base = (long long)blockIdx.x * TEX_THREADS + (threadIdx.x & ~31); base < d.total; base += stride) {
        const long long g = base + lane;
        // The trilinear lookup is formed once, before the channel loop.  The bilinear one (a single pass) is formed
        // inside the branch on g: that order takes fewer registers.
        Lookup q;
        q.t0.valid = false;
        if (MIP && g < d.total) q = lookup_of<MIP, VEC>(texture, pyramid, indices, derivatives, d, C, L, g);
        for (int c0 = 0; c0 < C; c0 += NV) {
            float v[NV];
#pragma unroll
            for (int j = 0; j < NV; ++j) v[j] = 0.f;
            if (MIP || g < d.total) {
                if (!MIP) q = lookup_of<MIP, VEC>(texture, pyramid, indices, derivatives, d, C, L, g);
                if (q.t0.valid) {
                    level_rows<NV, VEC>(q.p0, q.t0, q.w0, C, c0, !MIP && d.mode == DIRT_TEXTURE_NEAREST, v);
                    if (MIP && q.lod.f != 0.f) {
                        float u[NV];
                        level_rows<NV, VEC>(q.p1, q.t1, q.w1, C, c0, false, u);
                        const float omf = __fsub_rn(1.0f, q.lod.f);
#pragma unroll
                        for (int j = 0; j < NV; ++j) v[j] = __fadd_rn(__fmul_rn(omf, v[j]), __fmul_rn(q.lod.f, u[j]));
                    }
                }
            }
            store_out<CT, VEC>(out, stage, base, c0, C, d.total, v);
        }
    }
}

// Any C: one thread per output element (lookup g, channel c), so that loads of a texel's channels and the stores are
// coalesced.  The grid-stride step is precomputed as (step_g lookups, step_c channels).
__global__ void __launch_bounds__(TEX_THREADS) texture_forward_generic_kernel(const float* __restrict__ texture,
                                                                              const float* __restrict__ indices,
                                                                              float* __restrict__ out, TexDims d,
                                                                              long long step_g, int step_c)
{
    const long long e = (long long)blockIdx.x * TEX_THREADS + threadIdx.x;
    long long g = e / d.C;
    int c = (int)(e - g * d.C);
    const int C = d.C;
    while (g < d.total) {
        float v = 0.f;
        const float ir = __ldg(indices + 2 * g), ic = __ldg(indices + 2 * g + 1);
        const Taps t = taps_of(ir, ic, d, g);
        if (t.valid) {
            const float* tex = texture + t.base * C + c;
            const float t00 = __ldg(tex + ((long long)t.r0 * d.TW + t.c0) * C);
            if (d.mode == DIRT_TEXTURE_NEAREST) {
                v = t00;
            } else {
                const float t01 = __ldg(tex + ((long long)t.r0 * d.TW + t.c1) * C);
                const float t10 = __ldg(tex + ((long long)t.r1 * d.TW + t.c0) * C);
                const float t11 = __ldg(tex + ((long long)t.r1 * d.TW + t.c1) * C);
                v = bilinear(t00, t01, t10, t11, t.fr, t.fc);
            }
        }
        out[g * C + c] = v;
        g += step_g;
        c += step_c;
        if (c >= C) { c -= C; ++g; }
    }
}

// ---- backward -------------------------------------------------------------------------------------------------------

// warp aggregation (Agg, agg_plan, agg_sum) and the vector reductions: common.cuh

template <int NV, bool VEC>
__device__ __forceinline__ void red_row(float* dst, const float v[NV])
{
    if (VEC && NV == 4) {
        red_add_v4(dst, v[0], v[1 % NV], v[2 % NV], v[3 % NV]);
    } else if (VEC && NV == 2) {
        red_add_v2(dst, v[0], v[1 % NV]);
    } else {
#pragma unroll
        for (int j = 0; j < NV; ++j) atomicAdd(dst + j, v[j]);
    }
}

// d out / d (row, col) index at one level, through the fractions only, added to (dr, dc): the level's taps t
// (omr = 1 - t.fr, omc = 1 - t.fc) in its texture tex of width TW.  go: grad_out's row (CT = 0: its channels are read
// one at a time into go[0]).
template <int CT, bool VEC>
__device__ __forceinline__ void index_grad_level(const float* tex, const Taps& t, float omr, float omc, int TW, int C,
                                                 const float* gout, float go[], float& dr, float& dc)
{
    constexpr int NV = CT ? CT : 1;
    const float* p00 = tex + ((long long)t.r0 * TW + t.c0) * C;
    const float* p01 = tex + ((long long)t.r0 * TW + t.c1) * C;
    const float* p10 = tex + ((long long)t.r1 * TW + t.c0) * C;
    const float* p11 = tex + ((long long)t.r1 * TW + t.c1) * C;
    for (int c0 = 0; c0 < C; c0 += NV) {
        float t00[NV], t01[NV], t10[NV], t11[NV];
        load_row<NV, VEC>(p00 + c0, t00);
        load_row<NV, VEC>(p01 + c0, t01);
        load_row<NV, VEC>(p10 + c0, t10);
        load_row<NV, VEC>(p11 + c0, t11);
        if (!CT) go[0] = __ldg(gout + c0);
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            dc += go[j] * ((t01[j] - t00[j]) * omr + (t11[j] - t10[j]) * t.fr);
            dr += go[j] * ((t10[j] - t00[j]) * omc + (t11[j] - t01[j]) * t.fc);
        }
    }
}

// d out / d texture at one level: the first `corners` bilinear weights of taps t (omr, omc as above; times the level
// weight a when MIP) scattered to the texels of dst (width TW, C channels), summed per texel in the warp with
// key_offset + the texel index as the key.  A level with t.valid false scatters nothing.  Warp-uniform: every lane
// takes part in agg_plan.
template <int CT, bool VEC, bool MIP>
__device__ __forceinline__ void texel_grad_level(const Taps& t, float omr, float omc, float a, long long key_offset,
                                                 float* dst_level, int TW, int C, int corners, const float go[],
                                                 const float* gout, int lane)
{
    constexpr int NV = CT ? CT : 1;
    for (int k = 0; k < corners; ++k) {   // (r0,c0), (r0,c1), (r1,c0), (r1,c1)
        const int r = (k & 2) ? t.r1 : t.r0, c = (k & 1) ? t.c1 : t.c0;
        float w = __fmul_rn((k & 1) ? t.fc : omc, (k & 2) ? t.fr : omr);
        if (MIP) w = __fmul_rn(w, a);
        const bool on = t.valid && w != 0.f;
        const long long texel = t.base + (long long)r * TW + c;
        // texel indices stay below 2^62 (checked in api.cu): bit 63 marks a lane's private key
        const Agg ag = agg_plan(on ? (unsigned long long)(key_offset + texel) : (1ull << 63) | (unsigned)lane, lane);
        const bool leader = on && __ffs(ag.peers) - 1 == lane;
        float* dst = dst_level + texel * C;
        if (CT) {
            float v[NV];
#pragma unroll
            for (int j = 0; j < NV; ++j) v[j] = on ? go[j] * w : 0.f;
            agg_sum<NV>(ag, v, lane);
            if (leader) red_row<NV, VEC>(dst, v);
        } else {
            for (int ch = 0; ch < C; ++ch) {
                float v[1] = {on ? __ldg(gout + ch) * w : 0.f};
                agg_sum<1>(ag, v, lane);
                if (leader) atomicAdd(dst + ch, v[0]);
            }
        }
    }
}

// One thread per lookup.  CT = C in 1..4, or 0 for any C (channels in a loop).  VEC: as in the forward kernel, for
// indices, derivatives, grad_indices, grad_out, and the rows of texture, pyramid, grad_texture and level_grad.
// MIP: grad_indices through both levels' fractions, each scaled by 2^-k.  The texel gradients of level 0 go to
// grad_texture, those of level k >= 1 to level_grad (the pyramid's layout), keyed on the packed texel index (level 0:
// its texel index; level k: TB * texels + the pyramid's texel index).
template <int CT, bool VEC, bool MIP>
__global__ void __launch_bounds__(TEX_THREADS) texture_backward_kernel(
    const float* __restrict__ texture, const float* __restrict__ indices, const float* __restrict__ grad_out,
    float* __restrict__ grad_texture, float* __restrict__ grad_indices, TexDims d, const float* __restrict__ pyramid,
    const float* __restrict__ derivatives, float* __restrict__ level_grad, int L)
{
    constexpr int NV = CT ? CT : 1;   // channels held in registers at a time
    const int C = CT ? CT : d.C;
    const int lane = threadIdx.x & 31;
    const bool bilinear_mode = MIP || d.mode == DIRT_TEXTURE_BILINEAR;
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long base = (long long)blockIdx.x * TEX_THREADS + (threadIdx.x & ~31); base < d.total; base += stride) {
        const long long g = base + lane;
        const bool live = g < d.total;
        Lookup q;
        q.t0.valid = false;
        if (!MIP) { q.t0.base = 0; q.t0.r0 = q.t0.r1 = q.t0.c0 = q.t0.c1 = 0; q.t0.fr = q.t0.fc = 0.f; }
        q.lod.l = 0; q.lod.f = 0.f;
        if (live) q = lookup_of<MIP, VEC>(texture, pyramid, indices, derivatives, d, C, L, g);
        if (MIP && !q.t0.valid) {   // an invalid lookup's taps are zero and scatter nothing
            q.t0.r0 = q.t0.r1 = q.t0.c0 = q.t0.c1 = 0; q.t0.fr = q.t0.fc = 0.f; q.t0.base = 0;
            q.t1 = q.t0;
            q.lod.l = 0; q.lod.f = 0.f;
        }
        const float omr = __fsub_rn(1.0f, q.t0.fr), omc = __fsub_rn(1.0f, q.t0.fc);   // level l
        const bool both = MIP && q.t0.valid && q.lod.f != 0.f;
        const float omf = __fsub_rn(1.0f, q.lod.f);
        const float* gout = grad_out + g * C;
        float go[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) go[j] = 0.f;
        if (CT && q.t0.valid) load_row<NV, VEC>(gout, go);

        if (grad_indices && live) {
            float dr = 0.f, dc = 0.f;
            if (q.t0.valid && bilinear_mode)
                index_grad_level<CT, VEC>(MIP ? q.p0 : texture + q.t0.base * C, q.t0, omr, omc, q.w0, C, gout, go, dr, dc);
            if (MIP) {
                float dr1 = 0.f, dc1 = 0.f;
                if (both)
                    index_grad_level<CT, VEC>(q.p1, q.t1, __fsub_rn(1.0f, q.t1.fr), __fsub_rn(1.0f, q.t1.fc), q.w1, C, gout,
                                              go, dr1, dc1);
                // d index_k / d index = 2^-k
                const float s0 = __int_as_float((127 - q.lod.l) << 23), s1 = 0.5f * s0;
                dr = dr * s0;
                dc = dc * s0;
                if (both) {
                    dr = omf * dr + q.lod.f * (dr1 * s1);
                    dc = omf * dc + q.lod.f * (dc1 * s1);
                }
            }
            if (VEC) reinterpret_cast<float2*>(grad_indices)[g] = make_float2(dr, dc);
            else { grad_indices[2 * g] = dr; grad_indices[2 * g + 1] = dc; }
        }

        // d out / d texture: the bilinear weights (1 for nearest) scattered to the texels, summed per texel in the warp
        if (grad_texture) {
            if (MIP) {
#pragma unroll 1
                for (int s = 0; s < 2; ++s) {
                    const int k = q.lod.l + s;
                    Taps t = s ? q.t1 : q.t0;
                    t.valid = s ? both : q.t0.valid;
                    const long long key_offset = k == 0 ? 0ll : (long long)d.TB * d.texels + mip_offset(d, k);
                    float* dst_level = k == 0 ? grad_texture : level_grad + mip_offset(d, k) * C;
                    texel_grad_level<CT, VEC, true>(t, __fsub_rn(1.0f, t.fr), __fsub_rn(1.0f, t.fc),
                                                    s ? q.lod.f : (both ? omf : 1.0f), key_offset, dst_level,
                                                    s ? q.w1 : q.w0, C, 4, go, gout, lane);
                }
            } else {
                texel_grad_level<CT, VEC, false>(q.t0, omr, omc, 1.0f, 0, grad_texture, d.TW, C, bilinear_mode ? 4 : 1, go,
                                                 gout, lane);
            }
        }
    }
}

inline bool aligned(const void* p, int bytes) { return (uintptr_t)p % bytes == 0; }

inline unsigned blocks_for(long long work)
{
    const long long b = (work + TEX_THREADS - 1) / TEX_THREADS;
    return (unsigned)(b < TEX_MAX_BLOCKS ? b : TEX_MAX_BLOCKS);
}

// f(std::integral_constant<int, CT>()) with the kernels' channel parameter: CT = C for C in 1..4, else 0 (any C)
template <typename F>
cudaError_t with_ct(int C, F f)
{
    switch (C) {
        case 1: return f(std::integral_constant<int, 1>());
        case 2: return f(std::integral_constant<int, 2>());
        case 3: return f(std::integral_constant<int, 3>());
        case 4: return f(std::integral_constant<int, 4>());
        default: return f(std::integral_constant<int, 0>());
    }
}

// The vector path needs 8-byte index pairs, 16-byte derivatives, out rows aligned for the float2 / float4 stores (16
// bytes for the staged C = 3 store), and texture and pyramid rows for the float2 / float4 loads.  Bilinear and nearest
// with any C run the generic kernel.
template <int CT, bool MIP>
cudaError_t forward_ct(const float* texture, const float* pyramid, const float* indices, const float* derivatives,
                       float* out, const TexDims& d, int L, cudaStream_t stream)
{
    if constexpr (CT == 0 && !MIP) {
        const unsigned blocks = blocks_for(d.total * d.C);
        const long long step = (long long)blocks * TEX_THREADS;
        texture_forward_generic_kernel<<<blocks, TEX_THREADS, 0, stream>>>(texture, indices, out, d, step / d.C,
                                                                            (int)(step % d.C));
    } else {
        const int row = CT == 2 || CT == 4 ? 4 * CT : 4;
        auto kernel = texture_forward_kernel<CT, false, MIP>;
        if constexpr (CT != 0)   // any C has no vector path
            if (aligned(indices, 8) && aligned(out, CT == 3 ? 16 : row) && aligned(texture, row) &&
                (!MIP || (aligned(derivatives, 16) && aligned(pyramid, row))))
                kernel = texture_forward_kernel<CT, true, MIP>;
        kernel<<<blocks_for(d.total), TEX_THREADS, 0, stream>>>(texture, indices, out, d, pyramid, derivatives, L);
    }
    return launched();
}

// The vector path needs 8-byte index pairs and grad_indices pairs, 16-byte derivatives, and the rows of grad_out,
// texture, pyramid, grad_texture and level_grad aligned for float2 / float4.  For any C it serves the index pairs of
// the bilinear lookup alone.
template <int CT, bool MIP>
cudaError_t backward_ct(const float* texture, const float* pyramid, const float* indices, const float* derivatives,
                        const float* grad_out, float* grad_texture, float* level_grad, float* grad_indices,
                        const TexDims& d, int L, cudaStream_t stream)
{
    const int row = CT == 2 || CT == 4 ? 4 * CT : 4;
    auto kernel = texture_backward_kernel<CT, false, MIP>;
    if constexpr (CT != 0 || !MIP)
        if (aligned(indices, 8) && aligned(grad_indices, 8) && aligned(grad_out, row) && aligned(texture, row) &&
            aligned(grad_texture, row) &&
            (!MIP || (aligned(derivatives, 16) && aligned(pyramid, row) && aligned(level_grad, row))))
            kernel = texture_backward_kernel<CT, true, MIP>;
    kernel<<<blocks_for(d.total), TEX_THREADS, 0, stream>>>(texture, indices, grad_out, grad_texture, grad_indices, d,
                                                            pyramid, derivatives, level_grad, L);
    return launched();
}

// ---- deterministic backward (DESIGN.md §7.5) ------------------------------------------------------------------------
//
// grad_texture with no float atomics: each (texel, channel) is one float64 sum in a fixed order, rounded once to fp32.
//  (1) A stable LSD radix sort of (key, id) over the lookups, 8 bits per pass and only as many passes as the largest key
//      needs.  A valid lookup's key is its base texel tb*TH*TW + r0*TW + c0, an invalid one's the sentinel TB*TH*TW; the
//      ids are the lookup ids g = b*N + n.  The first pass computes the keys from the indices (taps_of) and takes the
//      ids from the positions.  Per pass: a histogram per tile of RS_TILE lookups, an exclusive scan of each digit's
//      row of the [digit][tile] count matrix (one CTA per digit), and a scatter in which a lookup's rank in its tile
//      comes from MATCH.ANY on the digit and the warps' digit counts taken in warp order.  The output is unique.
//  (2) offsets[k] = the first sorted position whose key is >= k, k = 0 .. sentinel + 1, by binary search: the lookups
//      whose base is texel x are the segment [offsets[x], offsets[x + 1]).
//  (3) Texel x = (tb, r, c) receives the terms of four segments, in this order: corner 00 of base (r, c), corner 01 of
//      base (r, c-1), corner 10 of base (r-1, c), corner 11 of base (r-1, c-1), modulo the texture (nearest: corner 00
//      only).  A term is the fp32 product grad_out[g][ch] * w of the default kernel, w the corner's bilinear weight (a
//      zero weight gives +0.0), widened to float64.  The sequence's L terms are cut into chunks of DET_CHUNK; in chunk q
//      lane t of a warp sums the terms q*DET_CHUNK + t, + t + 32, ... in order from +0.0, the lanes meet in the xor
//      butterfly 16, 8, 4, 2, 1, and the chunk sums are added in chunk order from +0.0.  The tree depends on L alone.
//      A texel of at most DET_CHUNK terms is summed by one warp; a longer one is listed, each of its chunks is summed by
//      a warp of its own into the scratch, and one thread per (texel, channel) adds its chunks.
constexpr long long DET_CHUNK = 4096;       // terms per chunk of a texel's sum
#ifndef DIRT_TEX_DET_GRID
#define DIRT_TEX_DET_GRID 8192
#endif
constexpr unsigned DET_GRID = DIRT_TEX_DET_GRID;   // CTAs of the grid-stride passes

// the sort key of lookup g: its base texel, or the sentinel for an invalid lookup
struct LookupKey {
    const float* indices;
    TexDims d;
    unsigned sentinel;
    __device__ __forceinline__ unsigned operator()(long long g) const
    {
        const Taps t = taps_of(__ldg(indices + 2 * g), __ldg(indices + 2 * g + 1), d, g);
        return t.valid ? (unsigned)(t.base + (long long)t.r0 * d.TW + t.c0) : sentinel;
    }
};

// The term sequence of one texel: segment k (corner k) starts at sorted position s_k and holds terms [e_k, e_{k+1}) of
// the sequence (e_0 = 0, e_4 = L).  Scalars, not arrays, so that nothing is indexed dynamically.
struct TexSeq {
    int s0, s1, s2, s3;
    long long e1, e2, e3, L;
};

__device__ __forceinline__ TexSeq texel_sequence(const int* __restrict__ offsets, const TexDims& d, int x)
{
    const long long tb = x / d.texels, rc = x - tb * d.texels;
    const int r = (int)(rc / d.TW), c = (int)(rc - (long long)r * d.TW);
    const int rm = r == 0 ? d.TH - 1 : r - 1, cm = c == 0 ? d.TW - 1 : c - 1;
    const long long t0 = tb * d.texels;
    TexSeq q;
    const long long k0 = t0 + (long long)r * d.TW + c;
    q.s0 = __ldg(offsets + k0);
    q.e1 = __ldg(offsets + k0 + 1) - q.s0;
    if (d.mode == DIRT_TEXTURE_NEAREST) {
        q.s1 = q.s2 = q.s3 = 0;
        q.e2 = q.e3 = q.L = q.e1;
        return q;
    }
    const long long k1 = t0 + (long long)r * d.TW + cm, k2 = t0 + (long long)rm * d.TW + c, k3 = t0 + (long long)rm * d.TW + cm;
    q.s1 = __ldg(offsets + k1);
    q.e2 = q.e1 + (__ldg(offsets + k1 + 1) - q.s1);
    q.s2 = __ldg(offsets + k2);
    q.e3 = q.e2 + (__ldg(offsets + k2 + 1) - q.s2);
    q.s3 = __ldg(offsets + k3);
    q.L = q.e3 + (__ldg(offsets + k3 + 1) - q.s3);
    return q;
}

// Lane `lane`'s sums of terms i0 + lane, i0 + lane + 32, ... < i1 of the sequence, channels c0 .. c0 + NV - 1, then
// the warp's xor butterfly: every lane returns the chunk's sums.  Warp-uniform.
template <int NV>
__device__ __forceinline__ void chunk_sums(const TexSeq& q, long long i0, long long i1, int c0, const int* __restrict__ ids,
                                           const float* __restrict__ indices, const float* __restrict__ grad_out,
                                           const TexDims& d, int C, double acc[NV])
{
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int j = 0; j < NV; ++j) acc[j] = 0.0;
    for (long long i = i0 + lane; i < i1; i += 32) {
        const int k = i < q.e1 ? 0 : i < q.e2 ? 1 : i < q.e3 ? 2 : 3;
        const long long pos = k == 0 ? q.s0 + i : k == 1 ? q.s1 + (i - q.e1) : k == 2 ? q.s2 + (i - q.e2) : q.s3 + (i - q.e3);
        const long long g = __ldg(ids + pos);
        const Taps t = taps_of(__ldg(indices + 2 * g), __ldg(indices + 2 * g + 1), d, g);
        const float w = __fmul_rn((k & 1) ? t.fc : __fsub_rn(1.0f, t.fc), (k & 2) ? t.fr : __fsub_rn(1.0f, t.fr));
        const float* go = grad_out + g * C + c0;
#pragma unroll
        for (int j = 0; j < NV; ++j) acc[j] = __dadd_rn(acc[j], w != 0.f ? (double)__fmul_rn(__ldg(go + j), w) : 0.0);
    }
#pragma unroll
    for (int j = 0; j < NV; ++j)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[j] = __dadd_rn(acc[j], __shfl_xor_sync(FULL, acc[j], o));
}

struct TexDetArgs {
    const float *indices, *grad_out;
    const int *ids, *offsets;
    float* grad_texture;
    int* counters;        // [0] chunk slots taken, [1] long texels listed
    int4* long_list;      // (texel, first slot, chunks)
    int2* owner;          // per slot: (texel, chunk)
    double* partial;      // per slot: C chunk sums
    TexDims d;
};

// One warp per texel (CT = C in 1..4, or 0: any C, one channel at a time): a texel of at most DET_CHUNK terms is summed
// and written; a longer one takes slots for its chunks and is listed.
// (__maxnreg__ instead of __launch_bounds__: under the latter ptxas keeps the CT = 0 instance at 32 registers and spills)
template <int CT>
__global__ void __maxnreg__(64) tex_det_gather_kernel(TexDetArgs a)
{
    constexpr int NV = CT ? CT : 1;
    const int C = CT ? CT : a.d.C;
    const int lane = threadIdx.x & 31;
    const long long texels = (long long)a.d.TB * a.d.texels, warps = (long long)gridDim.x * (TEX_THREADS / 32);
    for (long long x = (long long)blockIdx.x * (TEX_THREADS / 32) + (threadIdx.x >> 5); x < texels; x += warps) {
        const TexSeq q = texel_sequence(a.offsets, a.d, (int)x);
        if (q.L > DET_CHUNK) {
            const int n = (int)((q.L + DET_CHUNK - 1) / DET_CHUNK);
            int slot = 0;
            if (lane == 0) {
                slot = atomicAdd(a.counters, n);
                a.long_list[atomicAdd(a.counters + 1, 1)] = make_int4((int)x, slot, n, 0);
            }
            slot = __shfl_sync(FULL, slot, 0);
            for (int c = lane; c < n; c += 32) a.owner[slot + c] = make_int2((int)x, c);
            continue;
        }
#pragma unroll 1
        for (int c0 = 0; c0 < C; c0 += NV) {
            double acc[NV];
            chunk_sums<NV>(q, 0, q.L, c0, a.ids, a.indices, a.grad_out, a.d, C, acc);
            if (lane == 0)
#pragma unroll
                for (int j = 0; j < NV; ++j) a.grad_texture[x * C + c0 + j] = __double2float_rn(__dadd_rn(0.0, acc[j]));
        }
    }
}

// one warp per chunk of a listed texel: its sums go to the chunk's slot
template <int CT>
__global__ void __launch_bounds__(TEX_THREADS) tex_det_chunk_kernel(TexDetArgs a)
{
    constexpr int NV = CT ? CT : 1;
    const int C = CT ? CT : a.d.C;
    const int lane = threadIdx.x & 31, slots = a.counters[0];
    const int warps = gridDim.x * (TEX_THREADS / 32);
    for (int s = blockIdx.x * (TEX_THREADS / 32) + (threadIdx.x >> 5); s < slots; s += warps) {
        const int2 o = a.owner[s];
        const TexSeq q = texel_sequence(a.offsets, a.d, o.x);
        const long long i0 = o.y * DET_CHUNK, i1 = i0 + DET_CHUNK < q.L ? i0 + DET_CHUNK : q.L;
        for (int c0 = 0; c0 < C; c0 += NV) {
            double acc[NV];
            chunk_sums<NV>(q, i0, i1, c0, a.ids, a.indices, a.grad_out, a.d, C, acc);
            if (lane == 0)
#pragma unroll
                for (int j = 0; j < NV; ++j) a.partial[(size_t)s * C + c0 + j] = acc[j];
        }
    }
}

// one thread per (listed texel, channel): the chunk sums in chunk order
__global__ void __launch_bounds__(TEX_THREADS) tex_det_finish_kernel(TexDetArgs a)
{
    const int C = a.d.C;
    const long long n = (long long)a.counters[1] * C, stride = (long long)gridDim.x * TEX_THREADS;
    for (long long e = (long long)blockIdx.x * TEX_THREADS + threadIdx.x; e < n; e += stride) {
        const int j = (int)(e / C), ch = (int)(e - (long long)j * C);
        const int4 t = a.long_list[j];
        double s = 0.0;
        for (int c = 0; c < t.z; ++c) s = __dadd_rn(s, a.partial[(size_t)(t.y + c) * C + ch]);
        a.grad_texture[(long long)t.x * C + ch] = __double2float_rn(s);
    }
}

template <int CT>
cudaError_t det_gather_ct(const TexDetArgs& a, unsigned gather_blocks, unsigned chunk_blocks, cudaStream_t stream)
{
    tex_det_gather_kernel<CT><<<gather_blocks, TEX_THREADS, 0, stream>>>(a);
    cudaError_t e = launched();
    if (e != cudaSuccess) return e;
    tex_det_chunk_kernel<CT><<<chunk_blocks, TEX_THREADS, 0, stream>>>(a);
    return launched();
}

inline unsigned det_blocks(long long work, long long per_block)
{
    const long long b = (work + per_block - 1) / per_block;
    return (unsigned)(b < 1 ? 1 : (b < DET_GRID ? b : DET_GRID));
}

}  // namespace

TexDetScratch carve_texture_det_scratch(void* base, const TexDims& d)
{
    TexDetScratch s = {};
    char* p = static_cast<char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char* r = p ? p + off : nullptr;
        off = align_up(off + bytes, 256);
        return r;
    };
    const size_t n = (size_t)d.total, texels = (size_t)d.TB * d.texels;
    const size_t tiles = (n + RS_TILE - 1) / RS_TILE;
    // a listed texel has more than DET_CHUNK terms, and there are n terms per corner
    const size_t terms = n * (d.mode == DIRT_TEXTURE_BILINEAR ? 4 : 1);
    const size_t max_long = terms / (DET_CHUNK + 1), max_slots = (terms + DET_CHUNK - 1) / DET_CHUNK + max_long;
    for (int k = 0; k < 2; ++k) s.keys[k] = reinterpret_cast<unsigned*>(take(n * sizeof(unsigned)));
    for (int k = 0; k < 2; ++k) s.ids[k] = reinterpret_cast<int*>(take(n * sizeof(int)));
    s.offsets = reinterpret_cast<int*>(take((texels + 2) * sizeof(int)));
    s.counts = reinterpret_cast<unsigned*>(take((size_t)RS_RADIX * tiles * sizeof(unsigned)));
    s.digit_total = reinterpret_cast<unsigned*>(take(RS_RADIX * sizeof(unsigned)));
    s.counters = reinterpret_cast<int*>(take(2 * sizeof(int)));
    s.long_list = reinterpret_cast<int4*>(take(max_long * sizeof(int4)));
    s.owner = reinterpret_cast<int2*>(take(max_slots * sizeof(int2)));
    s.partial = reinterpret_cast<double*>(take(max_slots * d.C * sizeof(double)));
    s.bytes = off;
    return s;
}

cudaError_t launch_texture_backward_deterministic(const float* texture, const float* indices, const float* grad_out,
                                                  float* grad_texture, float* grad_indices, const TexDims& d,
                                                  const TexDetScratch& s, cudaStream_t stream)
{
    // grad_indices is per lookup and has no atomics: the default kernel writes it
    if (!grad_texture || d.total == 0) return launch_texture_backward(texture, indices, grad_out, grad_texture, grad_indices, d,
                                                                      stream);
    cudaError_t e;
    if (grad_indices && (e = launch_texture_backward(texture, indices, grad_out, nullptr, grad_indices, d, stream)) !=
                            cudaSuccess)
        return e;
    if ((e = cudaMemsetAsync(s.counters, 0, 2 * sizeof(int), stream)) != cudaSuccess) return e;
    const unsigned sentinel = (unsigned)(d.TB * d.texels);
    int last;
    if ((e = sort_by_key(LookupKey{indices, d, sentinel}, d.total, sentinel, s.keys, s.ids, s.counts, s.digit_total, stream,
                         &last)) != cudaSuccess)
        return e;
    const unsigned* keys = s.keys[last];
    tex_segment_bounds_kernel<<<det_blocks((long long)sentinel + 2, TEX_THREADS), TEX_THREADS, 0, stream>>>(keys, d.total,
                                                                                                           sentinel, s.offsets);
    if ((e = launched()) != cudaSuccess) return e;
    TexDetArgs a;
    a.indices = indices; a.grad_out = grad_out; a.ids = s.ids[last]; a.offsets = s.offsets;
    a.grad_texture = grad_texture; a.counters = s.counters; a.long_list = s.long_list; a.owner = s.owner;
    a.partial = s.partial; a.d = d;
    const unsigned gather_blocks = det_blocks(sentinel, TEX_THREADS / 32);
    const long long terms = d.total * (d.mode == DIRT_TEXTURE_BILINEAR ? 4 : 1);
    const unsigned chunk_blocks = det_blocks(2 * ((terms + DET_CHUNK - 1) / DET_CHUNK), TEX_THREADS / 32);
    switch (d.C) {
        case 1: e = det_gather_ct<1>(a, gather_blocks, chunk_blocks, stream); break;
        case 2: e = det_gather_ct<2>(a, gather_blocks, chunk_blocks, stream); break;
        case 3: e = det_gather_ct<3>(a, gather_blocks, chunk_blocks, stream); break;
        case 4: e = det_gather_ct<4>(a, gather_blocks, chunk_blocks, stream); break;
        default: e = det_gather_ct<0>(a, gather_blocks, chunk_blocks, stream);
    }
    if (e != cudaSuccess) return e;
    tex_det_finish_kernel<<<det_blocks((terms / (DET_CHUNK + 1) + 1) * d.C, TEX_THREADS), TEX_THREADS, 0, stream>>>(a);
    return launched();
}

cudaError_t launch_texture_forward(const float* texture, const float* indices, float* out, const TexDims& d,
                                   cudaStream_t stream)
{
    return with_ct(d.C, [&](auto ct) {
        return forward_ct<decltype(ct)::value, false>(texture, nullptr, indices, nullptr, out, d, 1, stream);
    });
}

cudaError_t launch_texture_backward(const float* texture, const float* indices, const float* grad_out, float* grad_texture,
                                    float* grad_indices, const TexDims& d, cudaStream_t stream)
{
    cudaError_t e;
    if (grad_texture &&
        (e = cudaMemsetAsync(grad_texture, 0, sizeof(float) * (size_t)d.TB * d.texels * d.C, stream)) != cudaSuccess)
        return e;
    if (d.total == 0 || (!grad_texture && !grad_indices)) return cudaSuccess;
    return with_ct(d.C, [&](auto ct) {
        return backward_ct<decltype(ct)::value, false>(texture, nullptr, indices, nullptr, grad_out, grad_texture, nullptr,
                                                        grad_indices, d, 1, stream);
    });
}

// ---- mipmapped (trilinear) lookup (DESIGN.md §7.6): the pyramid, its adjoint and the deterministic level terms ------

namespace {

// one thread per element of the next level: ((a + b) + (c + e)) * 0.25 of the 2x2 block, in that order
__global__ void __launch_bounds__(TEX_THREADS) mip_build_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                                long long n, int H, int W, int C)
{
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long e = (long long)blockIdx.x * TEX_THREADS + threadIdx.x; e < n; e += stride) {
        const long long x = e / C, row = x / W;   // row = tb * H + i
        const int c = (int)(e - x * C), j = (int)(x - row * W);
        const float* s = src + ((2 * row) * (2ll * W) + 2 * j) * C + c;
        const long long down = 2ll * W * C;
        const float a = __ldg(s), b = __ldg(s + C), cc = __ldg(s + down), ee = __ldg(s + down + C);
        dst[e] = __fmul_rn(__fadd_rn(__fadd_rn(a, b), __fadd_rn(cc, ee)), 0.25f);
    }
}

// The pyramid's adjoint: each level-k texel passes 0.25 x its gradient to its four children.  One thread per element
// (level-0 texel, channel): acc = g_{L-1}[ancestor], then acc = g_k[ancestor] + 0.25 * acc for k = L-2 .. 1, and
// grad_texture += 0.25 * acc, each operation rounded in that order.  A gather: no atomics.
__global__ void __launch_bounds__(TEX_THREADS) mip_collapse_kernel(float* __restrict__ grad_texture,
                                                                   const float* __restrict__ level_grad, TexDims d, int L)
{
    const long long n = (long long)d.TB * d.texels * d.C, stride = (long long)gridDim.x * TEX_THREADS;
    for (long long e = (long long)blockIdx.x * TEX_THREADS + threadIdx.x; e < n; e += stride) {
        const long long x = e / d.C, tb = x / d.texels, rc = x - tb * d.texels;
        const int ch = (int)(e - x * d.C), r = (int)(rc / d.TW), c = (int)(rc - (long long)r * d.TW);
        float acc = 0.f;
        for (int k = L - 1; k >= 1; --k) {
            const long long tw = d.TW >> k, texels = d.texels >> (2 * k);
            const float v = __ldg(level_grad + (mip_offset(d, k) + tb * texels + (long long)(r >> k) * tw + (c >> k)) * d.C + ch);
            acc = k == L - 1 ? v : __fadd_rn(v, __fmul_rn(0.25f, acc));
        }
        grad_texture[e] = __fadd_rn(grad_texture[e], __fmul_rn(0.25f, acc));
    }
}

// Deterministic path, per level k: the lookups' level-k index (NaN where level k is not read, which the §7.5 path
// skips) and grad_out times their weight of level k, fp32
__global__ void __launch_bounds__(TEX_THREADS) mip_level_terms_kernel(const float* __restrict__ indices,
                                                                      const float* __restrict__ derivatives,
                                                                      const float* __restrict__ grad_out, TexDims d, int L,
                                                                      int k, float* __restrict__ level_indices,
                                                                      float* __restrict__ level_grad_out)
{
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long g = (long long)blockIdx.x * TEX_THREADS + threadIdx.x; g < d.total; g += stride) {
        const float ir = __ldg(indices + 2 * g), ic = __ldg(indices + 2 * g + 1);
        const Lod lod = lod_of(load_derivatives<false>(derivatives, g), L);
        const bool valid = isfinite(ir) && isfinite(ic);
        const float a = lod.l == k ? (lod.f != 0.f ? __fsub_rn(1.0f, lod.f) : 1.0f) : lod.f;
        const bool reads = valid && (lod.l == k || (lod.l + 1 == k && lod.f != 0.f));
        const float nan = __int_as_float(0x7fc00000);
        level_indices[2 * g] = reads ? level_index(ir, k) : nan;
        level_indices[2 * g + 1] = reads ? level_index(ic, k) : nan;
        for (int ch = 0; ch < d.C; ++ch) level_grad_out[g * d.C + ch] = reads ? __fmul_rn(__ldg(grad_out + g * d.C + ch), a) : 0.f;
    }
}

}  // namespace

MipScratch carve_texture_mip_scratch(void* base, const TexDims& d, bool deterministic)
{
    MipScratch s = {};
    char* p = static_cast<char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char* r = p && bytes ? p + off : nullptr;
        off = align_up(off + bytes, 256);
        return r;
    };
    const int L = mip_levels(d.TH, d.TW);
    s.level_grad = reinterpret_cast<float*>(take((size_t)mip_pyramid_texels(d, L) * d.C * sizeof(float)));
    if (deterministic) {
        s.indices = reinterpret_cast<float*>(take((size_t)d.total * 2 * sizeof(float)));
        s.grad_out = reinterpret_cast<float*>(take((size_t)d.total * d.C * sizeof(float)));
        s.det = take(carve_texture_det_scratch(nullptr, d).bytes);
    }
    s.bytes = off;
    return s;
}

cudaError_t launch_texture_mip_build(const float* texture, float* pyramid, const TexDims& d, cudaStream_t stream)
{
    const int L = mip_levels(d.TH, d.TW);
    for (int k = 1; k < L; ++k) {
        const long long n = (long long)d.TB * (d.texels >> (2 * k)) * d.C;
        mip_build_kernel<<<blocks_for(n), TEX_THREADS, 0, stream>>>(level_base(texture, (const float*)pyramid, d, k - 1),
                                                                    pyramid + mip_offset(d, k) * d.C, n, d.TH >> k,
                                                                    d.TW >> k, d.C);
        const cudaError_t e = launched();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_texture_trilinear_forward(const float* texture, const float* pyramid, const float* indices,
                                             const float* derivatives, float* out, const TexDims& d, cudaStream_t stream)
{
    const int L = mip_levels(d.TH, d.TW);
    return with_ct(d.C, [&](auto ct) {
        return forward_ct<decltype(ct)::value, true>(texture, pyramid, indices, derivatives, out, d, L, stream);
    });
}

cudaError_t launch_texture_trilinear_backward(const float* texture, const float* pyramid, const float* indices,
                                              const float* derivatives, const float* grad_out, float* grad_texture,
                                              float* grad_indices, const TexDims& d, bool deterministic,
                                              const MipScratch& s, cudaStream_t stream)
{
    const int L = mip_levels(d.TH, d.TW);
    const size_t texture_bytes = sizeof(float) * (size_t)d.TB * d.texels * d.C;
    cudaError_t e;
    if (d.total == 0 || !grad_texture) deterministic = false;
    if (grad_texture && !deterministic) {
        if ((e = cudaMemsetAsync(grad_texture, 0, texture_bytes, stream)) != cudaSuccess) return e;
        if (L > 1 && d.total > 0 &&
            (e = cudaMemsetAsync(s.level_grad, 0, sizeof(float) * (size_t)mip_pyramid_texels(d, L) * d.C, stream)) !=
                cudaSuccess)
            return e;
    }
    if (d.total == 0 || (!grad_texture && !grad_indices)) return cudaSuccess;
    // the default kernel: both gradients, or under the deterministic flag grad_indices alone (it has no atomics)
    float* gt = deterministic ? nullptr : grad_texture;
    if (gt || grad_indices) {
        e = with_ct(d.C, [&](auto ct) {
            return backward_ct<decltype(ct)::value, true>(texture, pyramid, indices, derivatives, grad_out, gt, s.level_grad,
                                                           grad_indices, d, L, stream);
        });
        if (e != cudaSuccess) return e;
    }
    if (!grad_texture) return cudaSuccess;
    if (deterministic) {
        // level k's gradient, every texel written, by the §7.5 path over the lookups that read level k
        for (int k = 0; k < L; ++k) {
            mip_level_terms_kernel<<<blocks_for(d.total), TEX_THREADS, 0, stream>>>(indices, derivatives, grad_out, d, L, k,
                                                                                     s.indices, s.grad_out);
            if ((e = launched()) != cudaSuccess) return e;
            TexDims dk = d;
            dk.TH = d.TH >> k; dk.TW = d.TW >> k; dk.texels = d.texels >> (2 * k);
            float* gk = k == 0 ? grad_texture : s.level_grad + mip_offset(d, k) * d.C;
            if ((e = launch_texture_backward_deterministic(nullptr, s.indices, s.grad_out, gk, nullptr, dk,
                                                           carve_texture_det_scratch(s.det, dk), stream)) !=
                cudaSuccess)
                return e;
        }
    }
    if (L > 1) {
        mip_collapse_kernel<<<blocks_for((long long)d.TB * d.texels * d.C), TEX_THREADS, 0, stream>>>(grad_texture, s.level_grad,
                                                                                                      d, L);
        if ((e = launched()) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- seamless cube-map lookup (DESIGN.md §7.10) ---------------------------------------------------------------------
//
// A lookup selects a face by the direction's major axis and reads the face's padded copy (S + 2 square, a one-texel
// border from the adjacent faces) with the bilinear rule of texture_forward_kernel, so that a footprint across an edge
// blends the right texels.  The atlas of padded faces is built per call (cube_atlas_kernel); the backward pass scatters
// to an atlas-shaped gradient and folds it into the cube map in a fixed order (cube_adjoint_kernel).

namespace {

// Faces +X, -X, +Y, -Y, +Z, -Z are 0 .. 5: the major axis, ties to x over y over z by exact comparisons
template <typename T>
__host__ __device__ __forceinline__ int cube_face(T x, T y, T z)
{
    const T ax = x < 0 ? -x : x, ay = y < 0 ? -y : y, az = z < 0 ? -z : z;
    if (ax >= ay && ax >= az) return x > 0 ? 0 : 1;
    if (ay >= az) return y > 0 ? 2 : 3;
    return z > 0 ? 4 : 5;
}

// the OpenGL cube-map table: face f's sc, tc and |ma| (negations and |.| are exact)
template <typename T>
__host__ __device__ __forceinline__ void cube_axes(int f, T x, T y, T z, T& sc, T& tc, T& ma)
{
    switch (f) {
        case 0: sc = -z; tc = -y; ma = x; break;
        case 1: sc = z; tc = -y; ma = -x; break;
        case 2: sc = x; tc = z; ma = y; break;
        case 3: sc = x; tc = -z; ma = -y; break;
        case 4: sc = x; tc = -y; ma = z; break;
        default: sc = -x; tc = -y; ma = -z; break;
    }
}

struct CubeTexel {
    int f, r, c;
};

// The cube texel that border texel (i, j) of face f's padded face copies (exactly one of i, j outside 1 .. S): the
// texel holding the projection of the direction through the border texel's centre, in float64.  The projection never
// lies within 1 / (S + 1) of a texel edge, so float64 rounding cannot move it.
__device__ __forceinline__ CubeTexel border_source(int f, int i, int j, int S)
{
    const double sc = 2.0 * (j - 0.5) / S - 1.0, tc = 2.0 * (i - 0.5) / S - 1.0;
    double x, y, z;
    switch (f) {
        case 0: x = 1.0; y = -tc; z = -sc; break;
        case 1: x = -1.0; y = -tc; z = sc; break;
        case 2: x = sc; y = 1.0; z = tc; break;
        case 3: x = sc; y = -1.0; z = -tc; break;
        case 4: x = sc; y = -tc; z = 1.0; break;
        default: x = -sc; y = -tc; z = -1.0; break;
    }
    CubeTexel o;
    o.f = cube_face(x, y, z);
    double s2, t2, ma;
    cube_axes(o.f, x, y, z, s2, t2, ma);
    const double s = (s2 / ma + 1.0) * 0.5, t = (t2 / ma + 1.0) * 0.5;
    o.r = min(max((int)floor(t * S), 0), S - 1);
    o.c = min(max((int)floor(s * S), 0), S - 1);
    return o;
}

// padded texel (i, j) of face f, item tb, in the atlas (d: one face's block)
__device__ __forceinline__ long long atlas_texel(const TexDims& d, int f, long long tb, int i, int j)
{
    return (((long long)f * d.TB + tb) * d.TH + i) * d.TW + j;
}

// One thread per atlas element (face, item, i, j, channel): the face texel inside, the adjacent face's texel on an edge
// of the border, ((own corner + row neighbour) + column neighbour) / 3 at a corner, each operation rounded in that order.
__global__ void __launch_bounds__(TEX_THREADS) cube_atlas_kernel(const float* __restrict__ cubemap, float* __restrict__ atlas,
                                                                 TexDims d)
{
    const int S = d.TW - 2, P = d.TW, C = d.C;
    const long long n = 6ll * d.TB * d.texels * C, stride = (long long)gridDim.x * TEX_THREADS;
    for (long long e = (long long)blockIdx.x * TEX_THREADS + threadIdx.x; e < n; e += stride) {
        const long long x = e / C, fb = x / d.texels;   // fb = f * TB + tb
        const int ch = (int)(e - x * C), f = (int)(fb / d.TB), ij = (int)(x - fb * d.texels), i = ij / P, j = ij - i * P;
        const long long tb = fb - (long long)f * d.TB;
        const float* cube = cubemap + tb * 6 * S * (long long)S * C + ch;
        auto at = [&](CubeTexel t) { return __ldg(cube + (((long long)t.f * S + t.r) * S + t.c) * C); };
        const bool out_i = i == 0 || i == P - 1, out_j = j == 0 || j == P - 1;
        float v;
        if (!out_i && !out_j) {
            v = at(CubeTexel{f, i - 1, j - 1});
        } else if (out_i != out_j) {
            v = at(border_source(f, i, j, S));
        } else {
            const int ii = i == 0 ? 1 : S, jj = j == 0 ? 1 : S;
            const float own = at(CubeTexel{f, ii - 1, jj - 1}), row = at(border_source(f, i, jj, S)),
                        col = at(border_source(f, ii, j, S));
            v = __fdiv_rn(__fadd_rn(__fadd_rn(own, row), col), 3.0f);
        }
        atlas[e] = v;
    }
}

// The border's adjoint: one thread per cube-map element (item, face, r, c, channel) sums, in this order and rounded
// in fp32, the gradient of its own padded texel, then for each edge of its face it lies on (row 0, row S-1, column 0,
// column S-1) the gradient of the border texel of the adjacent face that copies it, followed by a third of the
// gradient of each corner of that face that reads this border texel, and last a third of the gradient of each corner
// of its own face whose own texel it is.  A gather: no atomics.
__global__ void __launch_bounds__(TEX_THREADS) cube_adjoint_kernel(const float* __restrict__ grad_atlas,
                                                                   float* __restrict__ grad_cubemap, TexDims d)
{
    const int S = d.TW - 2, P = d.TW, C = d.C;
    const long long n = 6ll * d.TB * S * S * C, stride = (long long)gridDim.x * TEX_THREADS;
    for (long long e = (long long)blockIdx.x * TEX_THREADS + threadIdx.x; e < n; e += stride) {
        const long long x = e / C, tf = x / ((long long)S * S);   // tf = tb * 6 + f
        const int ch = (int)(e - x * C), rc = (int)(x - tf * S * S), r = rc / S, c = rc - r * S, f = (int)(tf % 6);
        const long long tb = tf / 6;
        auto at = [&](int g, int i, int j) { return __ldg(grad_atlas + atlas_texel(d, g, tb, i, j) * C + ch); };
        float acc = at(f, r + 1, c + 1);
        if (r == 0 || r == S - 1 || c == 0 || c == S - 1) {
#pragma unroll 1
            for (int k = 0; k < 4; ++k) {
                if (!(k == 0 ? r == 0 : k == 1 ? r == S - 1 : k == 2 ? c == 0 : c == S - 1)) continue;
                // the neighbour across this edge, and among its own neighbours across its edges the border texel
                // (qi, qj) of its face that copies (f, r, c)
                const CubeTexel y = k < 2 ? border_source(f, k == 0 ? 0 : P - 1, c + 1, S)
                                          : border_source(f, r + 1, k == 2 ? 0 : P - 1, S);
#pragma unroll 1
                for (int m = 0; m < 4; ++m) {
                    if (!(m == 0 ? y.r == 0 : m == 1 ? y.r == S - 1 : m == 2 ? y.c == 0 : y.c == S - 1)) continue;
                    const int qi = m < 2 ? (m == 0 ? 0 : P - 1) : y.r + 1, qj = m < 2 ? y.c + 1 : (m == 2 ? 0 : P - 1);
                    const CubeTexel z = border_source(y.f, qi, qj, S);
                    if (z.f != f || z.r != r || z.c != c) continue;
                    acc = __fadd_rn(acc, at(y.f, qi, qj));
                    // the corners of face y.f beside (qi, qj) read it as their row or column neighbour
                    if (m < 2) {
                        if (qj == 1) acc = __fadd_rn(acc, __fdiv_rn(at(y.f, qi, 0), 3.0f));
                        if (qj == S) acc = __fadd_rn(acc, __fdiv_rn(at(y.f, qi, P - 1), 3.0f));
                    } else {
                        if (qi == 1) acc = __fadd_rn(acc, __fdiv_rn(at(y.f, 0, qj), 3.0f));
                        if (qi == S) acc = __fadd_rn(acc, __fdiv_rn(at(y.f, P - 1, qj), 3.0f));
                    }
                    break;
                }
            }
            // the corners of its own face whose own texel it is
            for (int k = 0; k < 4; ++k) {
                const int ci = k < 2 ? 0 : P - 1, cj = (k & 1) ? P - 1 : 0;
                if ((ci == 0 ? r == 0 : r == S - 1) && (cj == 0 ? c == 0 : c == S - 1))
                    acc = __fadd_rn(acc, __fdiv_rn(at(f, ci, cj), 3.0f));
            }
        }
        grad_cubemap[e] = acc;
    }
}

// A lookup on the atlas: taps of the padded face (base: the face's block of the lookup's item), and the face
// coordinates its direction gradient needs.
struct CubeLookup {
    Taps t;
    int face;
    float sc, tc, ma;   // the face's table entries, ma = |major component|
};

// (t * S - 0.5) + 1 and the like, each operation rounded in the order of tests/cubemap_restatement.py
__device__ __forceinline__ CubeLookup cube_lookup(const float v[3], const TexDims& d, long long g)
{
    CubeLookup q;
    Taps& t = q.t;
    t.r0 = t.r1 = t.c0 = t.c1 = 0;
    t.fr = t.fc = 0.f;
    t.base = 0;
    q.face = 0;
    q.sc = q.tc = 0.f;
    q.ma = 1.f;
    t.valid = isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]) && (v[0] != 0.f || v[1] != 0.f || v[2] != 0.f);
    if (!t.valid) return q;
    q.face = cube_face(v[0], v[1], v[2]);
    cube_axes(q.face, v[0], v[1], v[2], q.sc, q.tc, q.ma);
    const int S = d.TW - 2;
    const float Sf = (float)S;
    const float s = __fmul_rn(__fadd_rn(__fdiv_rn(q.sc, q.ma), 1.0f), 0.5f);
    const float tt = __fmul_rn(__fadd_rn(__fdiv_rn(q.tc, q.ma), 1.0f), 0.5f);
    const long long tb = d.TB == 1 ? 0ll : g / d.N;
    t.base = atlas_texel(d, q.face, tb, 0, 0);
    if (d.mode == DIRT_TEXTURE_NEAREST) {
        t.r0 = t.r1 = min(max((int)floorf(__fmul_rn(tt, Sf)), 0), S - 1) + 1;
        t.c0 = t.c1 = min(max((int)floorf(__fmul_rn(s, Sf)), 0), S - 1) + 1;
        return q;
    }
    const float pr = __fadd_rn(__fsub_rn(__fmul_rn(tt, Sf), 0.5f), 1.0f);
    const float pc = __fadd_rn(__fsub_rn(__fmul_rn(s, Sf), 0.5f), 1.0f);
    const float flr = floorf(pr), flc = floorf(pc);
    t.fr = __fsub_rn(pr, flr);
    t.fc = __fsub_rn(pc, flc);
    t.r0 = (int)flr;
    t.c0 = (int)flc;
    t.r1 = t.r0 + 1;
    t.c1 = t.c0 + 1;
    return q;
}

// ---- mipmapped (trilinear) cube-map lookup (DESIGN.md §7.11) ------------------------------------------------------
//
// Level k of a cube map of S texels per edge is the §7.6 box pyramid of each face, S >> k per edge, read with the
// bilinear rule above on its own padded faces.  The mip atlas packs the levels' atlases [6, TB, (S>>k)+2, (S>>k)+2, C]
// in level order; CubeMip::offset[k] is level k's first texel.  lod is given per lookup, in levels.

struct CubeMip {
    const float* lod;                     // [B*N] levels of detail
    int L;                                // levels
    long long offset[MIP_MAX_LEVELS];     // first texel of level k's atlas in the mip atlas
};

// the dims of level k's atlas, d those of level 0's
__host__ __device__ __forceinline__ TexDims cube_level_dims(const TexDims& d, int k)
{
    TexDims e = d;
    e.TW = e.TH = ((d.TW - 2) >> k) + 2;
    e.texels = (long long)e.TW * e.TW;
    return e;
}

// lambda = lod, NaN -> 0, clamped to [0, L-1]; l = floor(lambda), f = lambda - l
__device__ __forceinline__ Lod cube_lod_of(float x, int L)
{
    const float lam = isnan(x) ? 0.f : fminf(fmaxf(x, 0.f), (float)(L - 1));
    Lod o;
    o.l = (int)floorf(lam);
    o.f = __fsub_rn(lam, (float)o.l);
    return o;
}

// The two levels the backward pass reads, k0 = min(l, L-2) and k0 + 1 (both 0 when L = 1), and the forward's weights
// of each: (1-f, f) when f != 0, (1, 0) at level l < L-1, (0, 1) at l = L-1.  The difference of the two levels is
// d out / d lod.
struct CubeMipPair {
    int k0, k1;
    float a0, a1;
};

__device__ __forceinline__ CubeMipPair cube_mip_pair(const Lod& lod, int L)
{
    CubeMipPair p;
    if (L == 1) {
        p.k0 = p.k1 = 0;
        p.a0 = 1.f;
        p.a1 = 0.f;
    } else if (lod.l == L - 1) {
        p.k0 = L - 2;
        p.k1 = L - 1;
        p.a0 = 0.f;
        p.a1 = 1.f;
    } else {
        p.k0 = lod.l;
        p.k1 = lod.l + 1;
        p.a0 = lod.f != 0.f ? __fsub_rn(1.0f, lod.f) : 1.0f;
        p.a1 = lod.f;
    }
    return p;
}

// Per-CTA accumulation of the coarse levels in shared memory: the levels whose atlases (all six faces of one item)
// fit CUBE_SMEM_FLOATS floats together, from level L-1 downwards.  -DDIRT_CUBE_MIP_SMEM_FLOATS=0 turns it off (a
// budget, not one of the grid caps above).
#ifdef DIRT_CUBE_MIP_SMEM_FLOATS
constexpr int CUBE_SMEM_FLOATS = DIRT_CUBE_MIP_SMEM_FLOATS;
#else
constexpr int CUBE_SMEM_FLOATS = 6144;
#endif

// One thread per lookup, CT = C in 1..4 or 0 (any C, one channel at a time).  The 12-byte direction rows go through
// the warp's slice of shared memory; VEC: atlas and out rows aligned for the vector loads and stores (as forward_ct).
// MIP: the atlas is the mip atlas of m, and a lookup reads level l and, when f != 0, level l + 1.
template <int CT, bool VEC, bool MIP>
__global__ void __launch_bounds__(TEX_THREADS) cube_forward_kernel(const float* __restrict__ atlas,
                                                                   const float* __restrict__ directions,
                                                                   float* __restrict__ out, TexDims d, CubeMip m)
{
    constexpr int NV = CT ? CT : 1;
    const int C = CT ? CT : d.C;
    __shared__ __align__(16) float stage[TEX_THREADS * 3];
    float* s = stage + (threadIdx.x & ~31) * 3;
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long base = (long long)blockIdx.x * TEX_THREADS + (threadIdx.x & ~31); base < d.total; base += stride) {
        const long long g = base + lane;
        const int n = d.total - base < 32 ? (int)(d.total - base) : 32;
        float dir[3];
        stage_load<3>(directions, 3, base, n, s, lane, dir);
        Lod lod;
        lod.l = 0;
        lod.f = 0.f;
        if (MIP) lod = cube_lod_of(g < d.total ? __ldg(m.lod + g) : 0.f, m.L);
        const int l1 = lod.l + 1 < m.L ? lod.l + 1 : lod.l;
        const TexDims d0 = MIP ? cube_level_dims(d, lod.l) : d, d1 = cube_level_dims(d, l1);
        CubeLookup q = cube_lookup(dir, d0, g);
        CubeLookup q1;
        if (MIP) q1 = cube_lookup(dir, d1, g);
        if (g >= d.total) q.t.valid = false;
        for (int c0 = 0; c0 < C; c0 += NV) {
            float v[NV];
#pragma unroll
            for (int j = 0; j < NV; ++j) v[j] = 0.f;
            if (q.t.valid) {
                level_rows<NV, VEC>((MIP ? atlas + m.offset[lod.l] * C : atlas) + q.t.base * C, q.t, d0.TW, C, c0,
                                    !MIP && d.mode == DIRT_TEXTURE_NEAREST, v);
                if (MIP && lod.f != 0.f) {
                    float u[NV];
                    level_rows<NV, VEC>(atlas + (m.offset[l1] + q1.t.base) * C, q1.t, d1.TW, C, c0, false, u);
                    const float omf = __fsub_rn(1.0f, lod.f);
#pragma unroll
                    for (int j = 0; j < NV; ++j) v[j] = __fadd_rn(__fmul_rn(omf, v[j]), __fmul_rn(lod.f, u[j]));
                }
            }
            store_out<CT, VEC>(out, stage, base, c0, C, d.total, v);
        }
    }
}

// The shared-memory half of the coarse-level accumulation: the lookups' texel terms of levels >= first go to acc
// (level k's atlas at acc + (m.offset[k] - m.offset[first]) * C, one item's six faces) by shared-memory atomics; then
// flush adds every non-zero element to grad_atlas with one reduction per CTA and element.
struct CubeSmem {
    float* acc;     // NULL: no level is accumulated in shared memory
    int first;      // the first level accumulated there (L when none)
};

// d out / d texel of one lookup's taps t (weights times a) added to the level's accumulator acc (width TW, C
// channels) with shared-memory atomics; the products are texel_grad_level's
template <int CT>
__device__ __forceinline__ void texel_grad_smem(const Taps& t, float a, float* acc, int TW, int C, const float go[],
                                                const float* gout)
{
    constexpr int NV = CT ? CT : 1;
    const float omr = __fsub_rn(1.0f, t.fr), omc = __fsub_rn(1.0f, t.fc);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int r = (k & 2) ? t.r1 : t.r0, c = (k & 1) ? t.c1 : t.c0;
        const float w = __fmul_rn(__fmul_rn((k & 1) ? t.fc : omc, (k & 2) ? t.fr : omr), a);
        if (w == 0.f) continue;
        float* dst = acc + (t.base + (long long)r * TW + c) * C;
        if (CT) {
#pragma unroll
            for (int j = 0; j < NV; ++j) atomicAdd(dst + j, go[j] * w);
        } else {
            for (int ch = 0; ch < C; ++ch) atomicAdd(dst + ch, __ldg(gout + ch) * w);
        }
    }
}

__device__ __forceinline__ void cube_smem_flush(const CubeSmem& sm, const CubeMip& m, float* grad_atlas, int C)
{
    __syncthreads();
    const long long n = (m.offset[m.L] - m.offset[sm.first]) * C;
    float* dst = grad_atlas + m.offset[sm.first] * C;
    for (long long e = threadIdx.x; e < n; e += TEX_THREADS) {
        const float v = sm.acc[e];
        if (v != 0.f) atomicAdd(dst + e, v);
    }
}

// One thread per lookup: grad_directions through the fractions (index_grad_level, then the chain to the direction in
// registers), and the texel terms scattered to grad_atlas (texel_grad_level).  VEC: also grad_out and grad_atlas rows.
// MIP: the two levels of cube_mip_pair, grad_directions through both levels' fractions (d p / d t = S >> k at level
// k), grad_lod the difference of the two levels' values; the texel terms go to the levels' atlases in grad_atlas, or
// for the coarse levels of a CTA whose lookups share one cube map to shared memory first (CubeSmem).
template <int CT, bool VEC, bool MIP>
__global__ void __launch_bounds__(TEX_THREADS) cube_backward_kernel(const float* __restrict__ atlas,
                                                                    const float* __restrict__ directions,
                                                                    const float* __restrict__ grad_out,
                                                                    float* __restrict__ grad_atlas,
                                                                    float* __restrict__ grad_directions, TexDims d,
                                                                    CubeMip m, float* __restrict__ grad_lod, int smem_first)
{
    constexpr int NV = CT ? CT : 1;
    const int C = CT ? CT : d.C;
    __shared__ float stage[TEX_THREADS * 3];
    float* s = stage + (threadIdx.x & ~31) * 3;
    const int lane = threadIdx.x & 31;
    const bool bilinear_mode = d.mode == DIRT_TEXTURE_BILINEAR;
    CubeSmem sm;
    sm.acc = nullptr;
    sm.first = m.L;
    if (MIP && CUBE_SMEM_FLOATS > 0 && grad_atlas && smem_first < m.L) {
        extern __shared__ float cube_smem[];
        sm.acc = cube_smem;
        sm.first = smem_first;
        const long long n = (m.offset[m.L] - m.offset[sm.first]) * C;
        for (long long e = threadIdx.x; e < n; e += TEX_THREADS) sm.acc[e] = 0.f;
        __syncthreads();
    }
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long base = (long long)blockIdx.x * TEX_THREADS + (threadIdx.x & ~31); base < d.total; base += stride) {
        const long long g = base + lane;
        const bool live = g < d.total;
        const int n = d.total - base < 32 ? (int)(d.total - base) : 32;
        float dir[3];
        stage_load<3>(directions, 3, base, n, s, lane, dir);
        float x = 0.f;
        CubeMipPair p;
        p.k0 = p.k1 = 0;
        p.a0 = 1.f;
        p.a1 = 0.f;
        if (MIP) {
            x = live ? __ldg(m.lod + g) : 0.f;
            p = cube_mip_pair(cube_lod_of(x, m.L), m.L);
        }
        const TexDims d0 = MIP ? cube_level_dims(d, p.k0) : d, d1 = cube_level_dims(d, p.k1);
        CubeLookup q = cube_lookup(dir, d0, g);
        CubeLookup q1;
        if (MIP) q1 = cube_lookup(dir, d1, g);
        if (!live) q.t.valid = false;   // its taps are never used to address memory
        const float omr = __fsub_rn(1.0f, q.t.fr), omc = __fsub_rn(1.0f, q.t.fc);
        const float* gout = grad_out + g * C;
        const float* lev0 = MIP ? atlas + m.offset[p.k0] * C : atlas;
        const float* lev1 = atlas + m.offset[p.k1] * C;
        float go[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) go[j] = 0.f;
        if (CT && q.t.valid) load_row<NV, VEC>(gout, go);

        if (MIP && grad_lod) {
            // d out / d lod = sum_c grad_out_c (b_{k1,c} - b_{k0,c}); 0 where the clamp is active, for NaN and L = 1
            float gl = 0.f;
            if (q.t.valid && m.L > 1 && x >= 0.f && x <= (float)(m.L - 1)) {
                for (int c0 = 0; c0 < C; c0 += NV) {
                    float v[NV], u[NV];
                    level_rows<NV, VEC>(lev0 + q.t.base * C, q.t, d0.TW, C, c0, false, v);
                    level_rows<NV, VEC>(lev1 + q1.t.base * C, q1.t, d1.TW, C, c0, false, u);
#pragma unroll
                    for (int j = 0; j < NV; ++j) gl += (CT ? go[j] : __ldg(gout + c0)) * (u[j] - v[j]);
                }
            }
            if (live) grad_lod[g] = gl;
        }

        if (grad_directions) {
            float gd[3] = {0.f, 0.f, 0.f};
            if (q.t.valid && bilinear_mode) {
                float dr = 0.f, dc = 0.f;
                if (!MIP || p.a0 != 0.f) index_grad_level<CT, VEC>(lev0 + q.t.base * C, q.t, omr, omc, d0.TW, C, gout, go, dr, dc);
                if (MIP) {
                    // d p_k / d t = S >> k at level k, the levels blended by their weights
                    float dr1 = 0.f, dc1 = 0.f;
                    if (p.a1 != 0.f)
                        index_grad_level<CT, VEC>(lev1 + q1.t.base * C, q1.t, __fsub_rn(1.0f, q1.t.fr),
                                                  __fsub_rn(1.0f, q1.t.fc), d1.TW, C, gout, go, dr1, dc1);
                    const float s0 = (float)(d0.TW - 2), s1 = (float)(d1.TW - 2);
                    dr = p.a0 * (dr * s0) + p.a1 * (dr1 * s1);
                    dc = p.a0 * (dc * s0) + p.a1 * (dc1 * s1);
                }
                // s = (sc / ma + 1) / 2, t likewise, pc = s * S + 1/2, pr = t * S + 1/2
                const float h = 0.5f * (MIP ? 1.0f : (float)(d.TW - 2)) / q.ma;
                const float gsc = dc * h, gtc = dr * h, gma = -(gsc * q.sc + gtc * q.tc) / q.ma;
                switch (q.face) {
                    case 0: gd[0] = gma; gd[1] = -gtc; gd[2] = -gsc; break;
                    case 1: gd[0] = -gma; gd[1] = -gtc; gd[2] = gsc; break;
                    case 2: gd[0] = gsc; gd[1] = gma; gd[2] = gtc; break;
                    case 3: gd[0] = gsc; gd[1] = -gma; gd[2] = -gtc; break;
                    case 4: gd[0] = gsc; gd[1] = -gtc; gd[2] = gma; break;
                    default: gd[0] = -gsc; gd[1] = -gtc; gd[2] = -gma; break;
                }
            }
            stage_store<3>(grad_directions, base, n, s, lane, gd);
        }
        if (grad_atlas) {
            if (MIP) {
#pragma unroll 1
                for (int i = 0; i < 2; ++i) {
                    const int k = i ? p.k1 : p.k0;
                    Taps t = i ? q1.t : q.t;
                    const float a = i ? p.a1 : p.a0;
                    const bool on = q.t.valid && a != 0.f, shared = k >= sm.first;
                    if (on && shared)
                        texel_grad_smem<CT>(t, a, sm.acc + (m.offset[k] - m.offset[sm.first]) * C, i ? d1.TW : d0.TW, C,
                                            go, gout);
                    t.valid = on && !shared;
                    if (__any_sync(FULL, t.valid))   // warp-uniform: texel_grad_level is collective
                        texel_grad_level<CT, VEC, true>(t, __fsub_rn(1.0f, t.fr), __fsub_rn(1.0f, t.fc), a, m.offset[k],
                                                        grad_atlas + m.offset[k] * C, i ? d1.TW : d0.TW, C, 4, go, gout,
                                                        lane);
                }
            } else {
                texel_grad_level<CT, VEC, false>(q.t, omr, omc, 1.0f, 0, grad_atlas, d.TW, C, bilinear_mode ? 4 : 1, go,
                                                 gout, lane);
            }
        }
    }
    if (MIP && sm.acc) cube_smem_flush(sm, m, grad_atlas, C);
}

// Deterministic path, per face f: the padded (row, col) of the lookups on face f (whole numbers for nearest), NaN for
// the others and for invalid lookups, which the §7.5 path skips
__global__ void __launch_bounds__(TEX_THREADS) cube_face_indices_kernel(const float* __restrict__ directions, TexDims d,
                                                                        int f, float* __restrict__ face_indices)
{
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long g = (long long)blockIdx.x * TEX_THREADS + threadIdx.x; g < d.total; g += stride) {
        const float v[3] = {__ldg(directions + 3 * g), __ldg(directions + 3 * g + 1), __ldg(directions + 3 * g + 2)};
        const CubeLookup q = cube_lookup(v, d, g);
        const bool on = q.t.valid && q.face == f;
        const float nan = __int_as_float(0x7fc00000);
        // r0 + fr is the padded row pr exactly (pr - floor(pr) is exact), so the sorted path forms the same taps
        face_indices[2 * g] = on ? (float)q.t.r0 + q.t.fr : nan;
        face_indices[2 * g + 1] = on ? (float)q.t.c0 + q.t.fc : nan;
    }
}

// Deterministic mipmapped path, per level k and face f: the padded (row, col) at level k of the lookups on face f
// that read level k with a non-zero weight, NaN for the others (and invalid lookups), which the §7.5 path skips; with
// write_grad_out also grad_out times each lookup's weight of level k (0 where it does not read it), fp32
__global__ void __launch_bounds__(TEX_THREADS) cube_mip_terms_kernel(const float* __restrict__ directions, TexDims d,
                                                                     CubeMip m, const float* __restrict__ grad_out, int k,
                                                                     int f, bool write_grad_out,
                                                                     float* __restrict__ level_indices,
                                                                     float* __restrict__ level_grad_out)
{
    const TexDims dk = cube_level_dims(d, k);
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long g = (long long)blockIdx.x * TEX_THREADS + threadIdx.x; g < d.total; g += stride) {
        const float v[3] = {__ldg(directions + 3 * g), __ldg(directions + 3 * g + 1), __ldg(directions + 3 * g + 2)};
        const CubeMipPair p = cube_mip_pair(cube_lod_of(__ldg(m.lod + g), m.L), m.L);
        const float a = k == p.k0 ? p.a0 : k == p.k1 ? p.a1 : 0.f;
        const CubeLookup q = cube_lookup(v, dk, g);
        const bool on = q.t.valid && q.face == f && a != 0.f;
        const float nan = __int_as_float(0x7fc00000);
        level_indices[2 * g] = on ? (float)q.t.r0 + q.t.fr : nan;
        level_indices[2 * g + 1] = on ? (float)q.t.c0 + q.t.fc : nan;
        if (write_grad_out)
            for (int ch = 0; ch < d.C; ++ch) level_grad_out[g * d.C + ch] = __fmul_rn(__ldg(grad_out + g * d.C + ch), a);
    }
}

template <int CT, bool MIP>
cudaError_t cube_forward_ct(const float* atlas, const float* directions, float* out, const TexDims& d, const CubeMip& m,
                            cudaStream_t stream)
{
    const int row = CT == 2 || CT == 4 ? 4 * CT : 4;
    auto kernel = cube_forward_kernel<CT, false, MIP>;
    if constexpr (CT != 0)
        if (aligned(out, CT == 3 ? 16 : row) && aligned(atlas, row)) kernel = cube_forward_kernel<CT, true, MIP>;
    kernel<<<blocks_for(d.total), TEX_THREADS, 0, stream>>>(atlas, directions, out, d, m);
    return launched();
}

// MIP: the shared-memory levels (smem_first < m.L) take (offset[L] - offset[smem_first]) * C floats of dynamic shared
// memory, and the grid is capped at 8 CTAs per SM, so that each CTA flushes them once for many lookups
template <int CT, bool MIP>
cudaError_t cube_backward_ct(const float* atlas, const float* directions, const float* grad_out, float* grad_atlas,
                             float* grad_directions, const TexDims& d, const CubeMip& m, float* grad_lod, int smem_first,
                             cudaStream_t stream)
{
    const int row = CT == 2 || CT == 4 ? 4 * CT : 4;
    auto kernel = cube_backward_kernel<CT, false, MIP>;
    if constexpr (CT != 0)
        if (aligned(grad_out, row) && aligned(atlas, row) && aligned(grad_atlas, row))
            kernel = cube_backward_kernel<CT, true, MIP>;
    unsigned blocks = blocks_for(d.total);
    size_t smem = 0;
    if (MIP && grad_atlas && smem_first < m.L) {
        smem = sizeof(float) * (size_t)(m.offset[m.L] - m.offset[smem_first]) * d.C;
        int dev = 0, sms = 0;
        cudaError_t e;
        if ((e = cudaGetDevice(&dev)) != cudaSuccess ||
            (e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess)
            return e;
        blocks = blocks < 8u * sms ? blocks : 8u * sms;
    }
    kernel<<<blocks, TEX_THREADS, smem, stream>>>(atlas, directions, grad_out, grad_atlas, grad_directions, d, m, grad_lod,
                                                  smem_first);
    return launched();
}

// the mip atlas's levels: offset[k], k = 0 .. L, of level k's first texel
CubeMip cube_mip_of(const TexDims& d, const float* lod)
{
    CubeMip m = {};
    m.lod = lod;
    m.L = mip_levels(d.TW - 2, d.TW - 2);
    for (int k = 0; k < m.L; ++k) {
        const long long P = ((d.TW - 2) >> k) + 2;
        m.offset[k + 1] = m.offset[k] + 6ll * d.TB * P * P;
    }
    return m;
}

// the first level accumulated in shared memory: the coarsest levels whose atlases fit CUBE_SMEM_FLOATS together, for
// a shared cube map (every CTA's lookups read one item); L for none
int cube_smem_first(const TexDims& d, const CubeMip& m)
{
    int first = m.L;
    if (d.TB == 1)
        while (first > 0 && (m.offset[m.L] - m.offset[first - 1]) * d.C <= CUBE_SMEM_FLOATS) --first;
    return first;
}

}  // namespace

CubeScratch carve_cubemap_scratch(void* base, const TexDims& d, bool deterministic)
{
    CubeScratch s = {};
    char* p = static_cast<char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char* r = p && bytes ? p + off : nullptr;
        off = align_up(off + bytes, 256);
        return r;
    };
    s.grad_atlas = reinterpret_cast<float*>(take(6 * (size_t)d.TB * d.texels * d.C * sizeof(float)));
    if (deterministic) {
        s.indices = reinterpret_cast<float*>(take((size_t)d.total * 2 * sizeof(float)));
        s.det = take(carve_texture_det_scratch(nullptr, d).bytes);
    }
    s.bytes = off;
    return s;
}

cudaError_t launch_cubemap_forward(const float* cubemap, const float* directions, float* atlas, float* out,
                                   const TexDims& d, cudaStream_t stream)
{
    cube_atlas_kernel<<<blocks_for(6ll * d.TB * d.texels * d.C), TEX_THREADS, 0, stream>>>(cubemap, atlas, d);
    const cudaError_t e = launched();
    if (e != cudaSuccess || d.total == 0) return e;
    return with_ct(d.C, [&](auto ct) {
        return cube_forward_ct<decltype(ct)::value, false>(atlas, directions, out, d, CubeMip{}, stream);
    });
}

cudaError_t launch_cubemap_backward(const float* atlas, const float* directions, const float* grad_out, float* grad_cubemap,
                                    float* grad_directions, const TexDims& d, bool deterministic, const CubeScratch& s,
                                    cudaStream_t stream)
{
    const int S = d.TW - 2;
    cudaError_t e;
    if (d.total == 0) {
        if (grad_cubemap &&
            (e = cudaMemsetAsync(grad_cubemap, 0, sizeof(float) * 6 * (size_t)d.TB * S * S * d.C, stream)) != cudaSuccess)
            return e;
        return cudaSuccess;
    }
    if (!grad_cubemap) deterministic = false;
    if (grad_cubemap && !deterministic &&
        (e = cudaMemsetAsync(s.grad_atlas, 0, sizeof(float) * 6 * (size_t)d.TB * d.texels * d.C, stream)) != cudaSuccess)
        return e;
    // the default kernel: both gradients, or under the deterministic flag grad_directions alone (it has no atomics)
    float* ga = grad_cubemap && !deterministic ? s.grad_atlas : nullptr;
    if (ga || grad_directions) {
        e = with_ct(d.C, [&](auto ct) {
            return cube_backward_ct<decltype(ct)::value, false>(atlas, directions, grad_out, ga, grad_directions, d,
                                                                 CubeMip{}, nullptr, 0, stream);
        });
        if (e != cudaSuccess) return e;
    }
    if (!grad_cubemap) return cudaSuccess;
    if (deterministic) {
        // face f's block of grad_atlas, every texel written, by the §7.5 path over the lookups on face f
        for (int f = 0; f < 6; ++f) {
            cube_face_indices_kernel<<<blocks_for(d.total), TEX_THREADS, 0, stream>>>(directions, d, f, s.indices);
            if ((e = launched()) != cudaSuccess) return e;
            if ((e = launch_texture_backward_deterministic(nullptr, s.indices, grad_out,
                                                           s.grad_atlas + (size_t)f * d.TB * d.texels * d.C, nullptr, d,
                                                           carve_texture_det_scratch(s.det, d), stream)) !=
                cudaSuccess)
                return e;
        }
    }
    cube_adjoint_kernel<<<blocks_for(6ll * d.TB * S * S * d.C), TEX_THREADS, 0, stream>>>(s.grad_atlas, grad_cubemap, d);
    return launched();
}

// ---- mipmapped cube-map lookup (DESIGN.md §7.11) ----

// the cube maps [TB, 6, S, S, C] as one texture of 6 * TB faces, the §7.6 pyramid's level 0
static TexDims cube_faces_dims(const TexDims& d)
{
    TexDims p = d;
    p.TB = 6 * d.TB;
    p.TH = p.TW = d.TW - 2;
    p.texels = (long long)p.TW * p.TW;
    p.total = 0;
    p.mode = DIRT_TEXTURE_BILINEAR;
    return p;
}

size_t cubemap_mip_atlas_texels(const TexDims& d) { return (size_t)cube_mip_of(d, nullptr).offset[mip_levels(d.TW - 2, d.TW - 2)]; }

CubeMipScratch carve_cubemap_mip_scratch(void* base, const TexDims& d, bool deterministic)
{
    CubeMipScratch s = {};
    char* p = static_cast<char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char* r = p && bytes ? p + off : nullptr;
        off = align_up(off + bytes, 256);
        return r;
    };
    const TexDims pd = cube_faces_dims(d);
    const int L = mip_levels(pd.TW, pd.TW);
    s.grad_atlas = reinterpret_cast<float*>(take(cubemap_mip_atlas_texels(d) * d.C * sizeof(float)));
    s.level_grad = reinterpret_cast<float*>(take((size_t)mip_pyramid_texels(pd, L) * d.C * sizeof(float)));
    if (deterministic) {
        s.indices = reinterpret_cast<float*>(take((size_t)d.total * 2 * sizeof(float)));
        s.grad_out = reinterpret_cast<float*>(take((size_t)d.total * d.C * sizeof(float)));
        s.det = take(carve_texture_det_scratch(nullptr, d).bytes);
    }
    s.bytes = off;
    return s;
}

// The pyramid is built in level 0's slot of the atlas (it holds 6 TB (S + 2)^2 texels, the pyramid fewer than
// 6 TB S^2 / 3), the atlases of levels 1 .. L-1 from it, and level 0's atlas last, over it.
// every level's atlas from level 0 (cubemap) and levels 1 .. L-1 (the pyramid layout at levels), coarsest first, then
// the lookups
static cudaError_t cube_mip_atlas_lookup(const float* cubemap, const float* levels, const float* directions,
                                         const float* lod, float* atlas, float* out, const TexDims& d, cudaStream_t stream)
{
    const TexDims pd = cube_faces_dims(d);
    const CubeMip m = cube_mip_of(d, lod);
    cudaError_t e;
    for (int k = m.L - 1; k >= 0; --k) {
        const TexDims dk = cube_level_dims(d, k);
        cube_atlas_kernel<<<blocks_for(6ll * d.TB * dk.texels * d.C), TEX_THREADS, 0, stream>>>(
            k == 0 ? cubemap : levels + mip_offset(pd, k) * d.C, atlas + m.offset[k] * d.C, dk);
        if ((e = launched()) != cudaSuccess) return e;
    }
    return with_ct(d.C, [&](auto ct) { return cube_forward_ct<decltype(ct)::value, true>(atlas, directions, out, d, m, stream); });
}

cudaError_t launch_cubemap_mip_forward(const float* cubemap, const float* directions, const float* lod, float* atlas,
                                       float* out, const TexDims& d, cudaStream_t stream)
{
    const cudaError_t e = launch_texture_mip_build(cubemap, atlas, cube_faces_dims(d), stream);
    if (e != cudaSuccess) return e;
    return cube_mip_atlas_lookup(cubemap, atlas, directions, lod, atlas, out, d, stream);
}

// the lookups' gradients, and the cube map's by level: level 0 to grad_cubemap, levels 1 .. L-1 to s.level_grad; *done
// when grad_cubemap is complete (no lookups, or no grad_cubemap)
static cudaError_t cube_mip_level_grads(const float* atlas, const float* directions, const float* lod,
                                        const float* grad_out, float* grad_cubemap, float* grad_directions, float* grad_lod,
                                        const TexDims& d, bool deterministic, const CubeMipScratch& s, cudaStream_t stream,
                                        bool* done)
{
    *done = true;
    const TexDims pd = cube_faces_dims(d);
    const CubeMip m = cube_mip_of(d, lod);
    cudaError_t e;
    if (d.total == 0) {
        if (grad_cubemap &&
            (e = cudaMemsetAsync(grad_cubemap, 0, sizeof(float) * (size_t)pd.TB * pd.texels * d.C, stream)) != cudaSuccess)
            return e;
        return cudaSuccess;
    }
    if (!grad_cubemap) deterministic = false;
    if (grad_cubemap && !deterministic &&
        (e = cudaMemsetAsync(s.grad_atlas, 0, sizeof(float) * m.offset[m.L] * d.C, stream)) != cudaSuccess)
        return e;
    // the default kernel: every gradient, or under the deterministic flag grad_directions and grad_lod (no atomics)
    float* ga = grad_cubemap && !deterministic ? s.grad_atlas : nullptr;
    if (ga || grad_directions || grad_lod) {
        const int smem_first = cube_smem_first(d, m);
        e = with_ct(d.C, [&](auto ct) {
            return cube_backward_ct<decltype(ct)::value, true>(atlas, directions, grad_out, ga, grad_directions, d, m,
                                                                grad_lod, smem_first, stream);
        });
        if (e != cudaSuccess) return e;
    }
    if (!grad_cubemap) return cudaSuccess;
    if (deterministic) {
        // block (k, f) of grad_atlas, every texel written, by the §7.5 path over the lookups that read level k on face f
        for (int k = 0; k < m.L; ++k) {
            const TexDims dk = cube_level_dims(d, k);
            for (int f = 0; f < 6; ++f) {
                cube_mip_terms_kernel<<<blocks_for(d.total), TEX_THREADS, 0, stream>>>(directions, d, m, grad_out, k, f, f == 0,
                                                                                        s.indices, s.grad_out);
                if ((e = launched()) != cudaSuccess) return e;
                float* gk = s.grad_atlas + (m.offset[k] + (size_t)f * d.TB * dk.texels) * d.C;
                if ((e = launch_texture_backward_deterministic(nullptr, s.indices, s.grad_out, gk, nullptr, dk,
                                                               carve_texture_det_scratch(s.det, dk), stream)) !=
                    cudaSuccess)
                    return e;
            }
        }
    }
    // each level's border adjoint into the pyramid's layout (level 0: grad_cubemap), then the pyramid's adjoint
    for (int k = 0; k < m.L; ++k) {
        const TexDims dk = cube_level_dims(d, k);
        const long long S = dk.TW - 2;
        cube_adjoint_kernel<<<blocks_for(6ll * d.TB * S * S * d.C), TEX_THREADS, 0, stream>>>(
            s.grad_atlas + m.offset[k] * d.C, k == 0 ? grad_cubemap : s.level_grad + mip_offset(pd, k) * d.C, dk);
        if ((e = launched()) != cudaSuccess) return e;
    }
    *done = false;
    return cudaSuccess;
}

cudaError_t launch_cubemap_mip_backward(const float* atlas, const float* directions, const float* lod, const float* grad_out,
                                        float* grad_cubemap, float* grad_directions, float* grad_lod, const TexDims& d,
                                        bool deterministic, const CubeMipScratch& s, cudaStream_t stream)
{
    const TexDims pd = cube_faces_dims(d);
    const CubeMip m = cube_mip_of(d, lod);
    bool done;
    cudaError_t e = cube_mip_level_grads(atlas, directions, lod, grad_out, grad_cubemap, grad_directions, grad_lod, d,
                                         deterministic, s, stream, &done);
    if (e != cudaSuccess || done) return e;
    if (m.L > 1) {
        mip_collapse_kernel<<<blocks_for((long long)pd.TB * pd.texels * d.C), TEX_THREADS, 0, stream>>>(grad_cubemap,
                                                                                                       s.level_grad, pd, m.L);
        if ((e = launched()) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- split-sum GGX lookup (DESIGN.md §7.12): §7.11's lookup on the GGX-prefiltered levels (ibl.cu) ----

CubeGgxScratch carve_cubemap_ggx_scratch(void* base, const TexDims& d, bool deterministic)
{
    CubeGgxScratch s = {};
    s.mip = carve_cubemap_mip_scratch(base, d, deterministic);
    const TexDims pd = cube_faces_dims(d);
    const size_t src = sizeof(float) * (size_t)mip_pyramid_texels(pd, mip_levels(pd.TW, pd.TW)) * d.C;
    s.src_grad = base && src ? reinterpret_cast<float*>(static_cast<char*>(base) + s.mip.bytes) : nullptr;
    s.bytes = align_up(s.mip.bytes + src, 256);
    return s;
}

cudaError_t launch_cubemap_ggx_forward(const float* cubemap, const float* directions, const float* lod, float* atlas,
                                       float* out, const TexDims& d, cudaStream_t stream)
{
    const cudaError_t e = launch_ggx_prefilter(cubemap, atlas, d, stream);
    if (e != cudaSuccess) return e;
    return cube_mip_atlas_lookup(cubemap, atlas + ggx_layout(d).levels, directions, lod, atlas, out, d, stream);
}

// the lookups' backward pass and border adjoints as §7.11's, then the prefilter's adjoint into the box levels (level 0
// straight into grad_cubemap) and the box pyramid's adjoint
cudaError_t launch_cubemap_ggx_backward(const float* atlas, const float* directions, const float* lod, const float* grad_out,
                                        float* grad_cubemap, float* grad_directions, float* grad_lod, const TexDims& d,
                                        bool deterministic, const CubeGgxScratch& s, cudaStream_t stream)
{
    const TexDims pd = cube_faces_dims(d);
    const int L = mip_levels(pd.TW, pd.TW);
    bool done;
    cudaError_t e = cube_mip_level_grads(atlas, directions, lod, grad_out, grad_cubemap, grad_directions, grad_lod, d,
                                         deterministic, s.mip, stream, &done);
    if (e != cudaSuccess || done || L == 1) return e;
    if ((e = cudaMemsetAsync(s.src_grad, 0, sizeof(float) * (size_t)mip_pyramid_texels(pd, L) * d.C, stream)) != cudaSuccess)
        return e;
    if ((e = launch_ggx_prefilter_adjoint(atlas, s.mip.level_grad, s.src_grad, grad_cubemap, d, stream)) != cudaSuccess)
        return e;
    mip_collapse_kernel<<<blocks_for((long long)pd.TB * pd.texels * d.C), TEX_THREADS, 0, stream>>>(grad_cubemap, s.src_grad,
                                                                                                   pd, L);
    return launched();
}

}  // namespace dirt
