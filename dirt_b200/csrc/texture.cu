// texture.cu -- differentiable texture lookup (dirt_texture_sample / dirt_texture_sample_backward): the bilinear and
// nearest lookups of the reference's textured sample, restated in torch by examples/textured.py:sample_texture, whose
// values the forward kernel reproduces bit for bit (DESIGN.md §7.1).
//
// Forward: one thread per lookup (C = 1..4) or per output element (any other C).  The index pair arrives as one 8-byte
// load, the four texels through the read-only path, and the output leaves in vector stores: float2 / float4 for C = 2 / 4,
// and for C = 3 the warp's 32 x 3 values are staged in shared memory and written as 24 float4.
// Backward: one thread per lookup.  grad_indices comes from the same four texels.  grad_texture is aggregated inside the
// warp before it touches global memory: lanes that hit the same texel (MATCH.ANY on its linear index) sum their
// contributions and the lowest of them issues one reduction (a vector RED for C = 2 / 4).
#include "../../include/dirt_b200.h"
#include "common.cuh"

namespace dirt {

namespace {

constexpr int TEX_THREADS = 256;
constexpr long long TEX_MAX_BLOCKS = 1 << 16;   // grid-stride loops beyond this
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

// the CT channels of one texel (or of one grad_out row) through the read-only path
template <int CT, bool VEC>
__device__ __forceinline__ void load_row(const float* p, float v[CT])
{
    if (VEC && CT == 4) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(p));
        v[0] = q.x; v[1 % CT] = q.y; v[2 % CT] = q.z; v[3 % CT] = q.w;
    } else if (VEC && CT == 2) {
        const float2 q = __ldg(reinterpret_cast<const float2*>(p));
        v[0] = q.x; v[1 % CT] = q.y;
    } else {
#pragma unroll
        for (int j = 0; j < CT; ++j) v[j] = __ldg(p + j);
    }
}

// examples/textured.py's expression, one IEEE-rounded operation at a time and in its order:
// t00*(1-fc)*(1-fr) + t01*fc*(1-fr) + t10*(1-fc)*fr + t11*fc*fr
__device__ __forceinline__ float bilinear(float t00, float t01, float t10, float t11, float fr, float fc)
{
    const float omr = __fsub_rn(1.0f, fr), omc = __fsub_rn(1.0f, fc);
    const float a = __fmul_rn(__fmul_rn(t00, omc), omr);
    const float b = __fmul_rn(__fmul_rn(t01, fc), omr);
    const float c = __fmul_rn(__fmul_rn(t10, omc), fr);
    const float e = __fmul_rn(__fmul_rn(t11, fc), fr);
    return __fadd_rn(__fadd_rn(__fadd_rn(a, b), c), e);
}

// ---- forward --------------------------------------------------------------------------------------------------------

// One thread per lookup, CT = C in 1..4.  VEC: the pointers are aligned for the vector loads and stores (see
// launch_texture_forward).  The loop runs per warp, so that the C = 3 staging sees all 32 lanes.
template <int CT, bool VEC>
__global__ void __launch_bounds__(TEX_THREADS) texture_forward_kernel(const float* __restrict__ texture,
                                                                      const float* __restrict__ indices,
                                                                      float* __restrict__ out, TexDims d)
{
    __shared__ __align__(16) float stage[CT == 3 ? TEX_THREADS * 3 : 1];
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long base = (long long)blockIdx.x * TEX_THREADS + (threadIdx.x & ~31); base < d.total; base += stride) {
        const long long g = base + lane;
        float v[CT];
#pragma unroll
        for (int j = 0; j < CT; ++j) v[j] = 0.f;
        if (g < d.total) {
            const float2 ix = load_index<VEC>(indices, g);
            const Taps t = taps_of(ix.x, ix.y, d, g);
            if (t.valid) {
                const float* tex = texture + t.base * CT;
                float t00[CT], t01[CT], t10[CT], t11[CT];
                load_row<CT, VEC>(tex + ((long long)t.r0 * d.TW + t.c0) * CT, t00);
                if (d.mode == DIRT_TEXTURE_NEAREST) {
#pragma unroll
                    for (int j = 0; j < CT; ++j) v[j] = t00[j];
                } else {
                    load_row<CT, VEC>(tex + ((long long)t.r0 * d.TW + t.c1) * CT, t01);
                    load_row<CT, VEC>(tex + ((long long)t.r1 * d.TW + t.c0) * CT, t10);
                    load_row<CT, VEC>(tex + ((long long)t.r1 * d.TW + t.c1) * CT, t11);
#pragma unroll
                    for (int j = 0; j < CT; ++j) v[j] = bilinear(t00[j], t01[j], t10[j], t11[j], t.fr, t.fc);
                }
            }
        }
        float* o = out + g * CT;
        if (VEC && CT == 4) {
            if (g < d.total) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1 % CT], v[2 % CT], v[3 % CT]);
        } else if (VEC && CT == 2) {
            if (g < d.total) *reinterpret_cast<float2*>(o) = make_float2(v[0], v[1 % CT]);
        } else if (VEC && CT == 3 && base + 32 <= d.total) {
            // the warp's 96 consecutive floats start on a 384-byte boundary: 24 float4 stores
            float* s = stage + (threadIdx.x & ~31) * 3;
#pragma unroll
            for (int j = 0; j < CT; ++j) s[lane * 3 + j] = v[j];
            __syncwarp();
            if (lane < 24) *reinterpret_cast<float4*>(out + base * 3 + lane * 4) = reinterpret_cast<const float4*>(s)[lane];
            __syncwarp();
        } else if (g < d.total) {
#pragma unroll
            for (int j = 0; j < CT; ++j) o[j] = v[j];
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

// How the lanes of a warp that share a key sum their values.  Lanes that contribute nothing carry a key of their own.
struct Agg {
    unsigned peers;     // lanes with this lane's key, this lane included
    unsigned leaders;   // the lowest lane of every group of two or more
    bool pull;          // each leader pulls its members one by one (else: one butterfly over the warp per group)
};

__device__ __forceinline__ Agg agg_plan(unsigned long long key, int lane)
{
    Agg a;
    a.peers = __match_any_sync(FULL, key);
    const unsigned size = __popc(a.peers);
    const bool leader = __ffs(a.peers) - 1 == lane;
    a.leaders = __ballot_sync(FULL, leader && size > 1);
    // pulling costs (largest group - 1) shuffle rounds, the butterflies 5 per group of two or more
    a.pull = __reduce_max_sync(FULL, size) - 1 <= 5u * __popc(a.leaders);
    return a;
}

// On return the lowest lane of each group holds the group's sum in v (other lanes: unspecified).  Warp-uniform.
template <int NV>
__device__ __forceinline__ void agg_sum(const Agg& a, float v[NV], int lane)
{
    if (!a.leaders) return;
    if (a.pull) {
        float s[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) s[j] = v[j];
        unsigned rest = __ffs(a.peers) - 1 == lane ? a.peers & (a.peers - 1) : 0u;
        while (__any_sync(FULL, rest)) {
            const int src = rest ? __ffs(rest) - 1 : lane;
#pragma unroll
            for (int j = 0; j < NV; ++j) {
                const float x = __shfl_sync(FULL, v[j], src);
                if (rest) s[j] += x;
            }
            rest &= rest - 1;
        }
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] = s[j];
    } else {
        float s[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) s[j] = v[j];
        for (unsigned todo = a.leaders; todo; todo &= todo - 1) {
            const int L = __ffs(todo) - 1;
            const bool member = (a.peers >> L) & 1u;
#pragma unroll
            for (int j = 0; j < NV; ++j) {
                float x = member ? v[j] : 0.f;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(FULL, x, o);
                if (lane == L) s[j] = x;
            }
        }
#pragma unroll
        for (int j = 0; j < NV; ++j) v[j] = s[j];
    }
}

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d)
{
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b)
{
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

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

// One thread per lookup.  CT = C in 1..4, or 0 for any C (channels in a loop).  VEC: as in the forward kernel, for
// indices, grad_indices, grad_out, texture and grad_texture rows.
template <int CT, bool VEC>
__global__ void __launch_bounds__(TEX_THREADS) texture_backward_kernel(const float* __restrict__ texture,
                                                                       const float* __restrict__ indices,
                                                                       const float* __restrict__ grad_out,
                                                                       float* __restrict__ grad_texture,
                                                                       float* __restrict__ grad_indices, TexDims d)
{
    constexpr int NV = CT ? CT : 1;   // channels held in registers at a time
    const int C = CT ? CT : d.C;
    const int lane = threadIdx.x & 31;
    const bool bilinear_mode = d.mode == DIRT_TEXTURE_BILINEAR;
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long base = (long long)blockIdx.x * TEX_THREADS + (threadIdx.x & ~31); base < d.total; base += stride) {
        const long long g = base + lane;
        const bool live = g < d.total;
        Taps t;
        t.valid = false; t.base = 0; t.r0 = t.r1 = t.c0 = t.c1 = 0; t.fr = t.fc = 0.f;
        if (live) {
            const float2 ix = load_index<VEC>(indices, g);
            t = taps_of(ix.x, ix.y, d, g);
        }
        const float omr = __fsub_rn(1.0f, t.fr), omc = __fsub_rn(1.0f, t.fc);
        const float* gout = grad_out + g * C;
        float go[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) go[j] = 0.f;
        if (CT && t.valid) load_row<NV, VEC>(gout, go);

        // d out / d (row, col) index, through the fractions only
        if (grad_indices && live) {
            float dr = 0.f, dc = 0.f;
            if (t.valid && bilinear_mode) {
                const float* tex = texture + t.base * C;
                const float* p00 = tex + ((long long)t.r0 * d.TW + t.c0) * C;
                const float* p01 = tex + ((long long)t.r0 * d.TW + t.c1) * C;
                const float* p10 = tex + ((long long)t.r1 * d.TW + t.c0) * C;
                const float* p11 = tex + ((long long)t.r1 * d.TW + t.c1) * C;
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
            if (VEC) reinterpret_cast<float2*>(grad_indices)[g] = make_float2(dr, dc);
            else { grad_indices[2 * g] = dr; grad_indices[2 * g + 1] = dc; }
        }

        // d out / d texture: the bilinear weights (1 for nearest) scattered to the texels, summed per texel in the warp
        if (grad_texture) {
            const int corners = bilinear_mode ? 4 : 1;
            for (int k = 0; k < corners; ++k) {   // (r0,c0), (r0,c1), (r1,c0), (r1,c1)
                const int r = (k & 2) ? t.r1 : t.r0, c = (k & 1) ? t.c1 : t.c0;
                const float w = __fmul_rn((k & 1) ? t.fc : omc, (k & 2) ? t.fr : omr);
                const bool on = t.valid && w != 0.f;
                const long long texel = t.base + (long long)r * d.TW + c;
                // texel indices stay below 2^62 (checked in api.cu): bit 63 marks a lane's private key
                const Agg a = agg_plan(on ? (unsigned long long)texel : (1ull << 63) | (unsigned)lane, lane);
                const bool leader = on && __ffs(a.peers) - 1 == lane;
                float* dst = grad_texture + texel * C;
                if (CT) {
                    float v[NV];
#pragma unroll
                    for (int j = 0; j < NV; ++j) v[j] = on ? go[j] * w : 0.f;
                    agg_sum<NV>(a, v, lane);
                    if (leader) red_row<NV, VEC>(dst, v);
                } else {
                    for (int ch = 0; ch < C; ++ch) {
                        float v[1] = {on ? __ldg(gout + ch) * w : 0.f};
                        agg_sum<1>(a, v, lane);
                        if (leader) atomicAdd(dst + ch, v[0]);
                    }
                }
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

template <int CT>
cudaError_t forward_ct(const float* texture, const float* indices, float* out, const TexDims& d, cudaStream_t stream)
{
    const int vec_bytes = CT == 3 ? 16 : 4 * CT;
    const bool vec = aligned(indices, 8) && aligned(out, vec_bytes) && (CT == 3 || aligned(texture, 4 * CT));
    const unsigned blocks = blocks_for(d.total);
    if (vec) texture_forward_kernel<CT, true><<<blocks, TEX_THREADS, 0, stream>>>(texture, indices, out, d);
    else texture_forward_kernel<CT, false><<<blocks, TEX_THREADS, 0, stream>>>(texture, indices, out, d);
    return cudaGetLastError();
}

template <int CT>
cudaError_t backward_ct(const float* texture, const float* indices, const float* grad_out, float* grad_texture,
                        float* grad_indices, const TexDims& d, cudaStream_t stream)
{
    const int row = CT == 2 || CT == 4 ? 4 * CT : 4;
    const bool vec = aligned(indices, 8) && aligned(grad_indices, 8) && aligned(grad_out, row) && aligned(texture, row) &&
                     aligned(grad_texture, row);
    const unsigned blocks = blocks_for(d.total);
    if (vec)
        texture_backward_kernel<CT, true><<<blocks, TEX_THREADS, 0, stream>>>(texture, indices, grad_out, grad_texture,
                                                                             grad_indices, d);
    else
        texture_backward_kernel<CT, false><<<blocks, TEX_THREADS, 0, stream>>>(texture, indices, grad_out, grad_texture,
                                                                              grad_indices, d);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_texture_forward(const float* texture, const float* indices, float* out, const TexDims& d,
                                   cudaStream_t stream, int* launches)
{
    cudaError_t e;
    switch (d.C) {
        case 1: e = forward_ct<1>(texture, indices, out, d, stream); break;
        case 2: e = forward_ct<2>(texture, indices, out, d, stream); break;
        case 3: e = forward_ct<3>(texture, indices, out, d, stream); break;
        case 4: e = forward_ct<4>(texture, indices, out, d, stream); break;
        default: {
            const unsigned blocks = blocks_for(d.total * d.C);
            const long long step = (long long)blocks * TEX_THREADS;
            texture_forward_generic_kernel<<<blocks, TEX_THREADS, 0, stream>>>(texture, indices, out, d, step / d.C,
                                                                                (int)(step % d.C));
            e = cudaGetLastError();
        }
    }
    if (e == cudaSuccess) ++*launches;
    return e;
}

cudaError_t launch_texture_backward(const float* texture, const float* indices, const float* grad_out, float* grad_texture,
                                    float* grad_indices, const TexDims& d, cudaStream_t stream, int* launches)
{
    cudaError_t e;
    if (grad_texture &&
        (e = cudaMemsetAsync(grad_texture, 0, sizeof(float) * (size_t)d.TB * d.texels * d.C, stream)) != cudaSuccess)
        return e;
    if (d.total == 0 || (!grad_texture && !grad_indices)) return cudaSuccess;
    switch (d.C) {
        case 1: e = backward_ct<1>(texture, indices, grad_out, grad_texture, grad_indices, d, stream); break;
        case 2: e = backward_ct<2>(texture, indices, grad_out, grad_texture, grad_indices, d, stream); break;
        case 3: e = backward_ct<3>(texture, indices, grad_out, grad_texture, grad_indices, d, stream); break;
        case 4: e = backward_ct<4>(texture, indices, grad_out, grad_texture, grad_indices, d, stream); break;
        default: e = backward_ct<0>(texture, indices, grad_out, grad_texture, grad_indices, d, stream);
    }
    if (e == cudaSuccess) ++*launches;
    return e;
}

}  // namespace dirt
