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
// Deterministic backward (dirt_texture_sample_backward_deterministic): a radix sort of the lookups by base texel, then
// fixed-order float64 sums per texel; see the section below and DESIGN.md §7.5.
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
constexpr int RS_THREADS = 256;             // sort CTA: one thread per digit value
constexpr int RS_RADIX = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_TILE = 4096;               // lookups per sort tile, 16 per thread
constexpr long long DET_CHUNK = 4096;       // terms per chunk of a texel's sum
constexpr unsigned DET_GRID = 8192;         // CTAs of the grid-stride passes

__device__ __forceinline__ unsigned lookup_key(const float* indices, const TexDims& d, long long g, unsigned sentinel)
{
    const Taps t = taps_of(__ldg(indices + 2 * g), __ldg(indices + 2 * g + 1), d, g);
    return t.valid ? (unsigned)(t.base + (long long)t.r0 * d.TW + t.c0) : sentinel;
}

// Exclusive scan of one value per thread over the RS_THREADS threads of the CTA; *total gets the sum.  Contains
// __syncthreads(); warp_sums is RS_WARPS words of shared memory.
__device__ __forceinline__ unsigned block_exclusive_scan(unsigned v, unsigned* warp_sums, unsigned* total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(FULL, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    unsigned before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < RS_WARPS; ++w) {
        const unsigned s = warp_sums[w];
        before += w < warp ? s : 0u;
        all += s;
    }
    __syncthreads();
    *total = all;
    return before + x - v;
}

// counts[digit][tile]: how many lookups of the tile have the digit (key >> shift) & 255
template <bool FIRST>
__global__ void __launch_bounds__(RS_THREADS) tex_sort_hist_kernel(const unsigned* __restrict__ keys,
                                                                   const float* __restrict__ indices, TexDims d,
                                                                   unsigned sentinel, int shift,
                                                                   unsigned* __restrict__ counts, int tiles)
{
    __shared__ unsigned hist[RS_RADIX];
    hist[threadIdx.x] = 0;
    __syncthreads();
    const long long first = (long long)blockIdx.x * RS_TILE;
    for (int j = 0; j < RS_TILE / RS_THREADS; ++j) {
        const long long i = first + j * RS_THREADS + threadIdx.x;
        if (i < d.total) {
            const unsigned key = FIRST ? lookup_key(indices, d, i, sentinel) : __ldg(keys + i);
            atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
    }
    __syncthreads();
    counts[(size_t)threadIdx.x * tiles + blockIdx.x] = hist[threadIdx.x];
}

// one CTA per digit: its row of tile counts becomes the exclusive prefix, in place; the row's sum goes to digit_total
__global__ void __launch_bounds__(RS_THREADS) tex_sort_scan_kernel(unsigned* __restrict__ counts,
                                                                   unsigned* __restrict__ digit_total, int tiles)
{
    __shared__ unsigned warp_sums[RS_WARPS];
    unsigned* row = counts + (size_t)blockIdx.x * tiles;
    unsigned carry = 0;
    for (int base = 0; base < tiles; base += RS_THREADS) {
        const int i = base + threadIdx.x;
        const unsigned v = i < tiles ? row[i] : 0u;
        unsigned total;
        const unsigned ex = block_exclusive_scan(v, warp_sums, &total);
        if (i < tiles) row[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) digit_total[blockIdx.x] = carry;
}

// Stable scatter of one tile.  Its lookups go in 16 rounds of RS_THREADS consecutive ones; in a round a lookup's slot is
// the tile's running slot of its digit, plus the lookups of the lower warps with that digit, plus its rank among its
// warp's lanes with that digit.  Thread dgt keeps the running slot of digit dgt.
template <bool FIRST>
__global__ void __launch_bounds__(RS_THREADS) tex_sort_scatter_kernel(const unsigned* __restrict__ keys_in,
                                                                      const int* __restrict__ ids_in,
                                                                      const float* __restrict__ indices, TexDims d,
                                                                      unsigned sentinel, int shift,
                                                                      const unsigned* __restrict__ counts,
                                                                      const unsigned* __restrict__ digit_total, int tiles,
                                                                      unsigned* __restrict__ keys_out,
                                                                      int* __restrict__ ids_out)
{
    __shared__ unsigned warp_sums[RS_WARPS];
    __shared__ unsigned wcount[RS_WARPS][RS_RADIX];
    __shared__ unsigned woff[RS_WARPS][RS_RADIX];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, dgt = threadIdx.x;
    unsigned all;
    // the lookups of the smaller digits, then those of digit dgt in the earlier tiles
    unsigned run = block_exclusive_scan(digit_total[dgt], warp_sums, &all) + counts[(size_t)dgt * tiles + blockIdx.x];
#pragma unroll
    for (int w = 0; w < RS_WARPS; ++w) wcount[w][dgt] = 0;
    __syncthreads();
    const long long first = (long long)blockIdx.x * RS_TILE;
    for (int j = 0; j < RS_TILE / RS_THREADS; ++j) {
        const long long i = first + j * RS_THREADS + threadIdx.x;
        const bool live = i < d.total;
        unsigned key = 0;
        int id = 0;
        if (live) {
            key = FIRST ? lookup_key(indices, d, i, sentinel) : __ldg(keys_in + i);
            id = FIRST ? (int)i : __ldg(ids_in + i);
        }
        const unsigned digit = live ? (key >> shift) & 255u : (unsigned)RS_RADIX;
        const unsigned peers = __match_any_sync(FULL, digit);
        const unsigned rank = __popc(peers & ((1u << lane) - 1u));
        if (live && rank == 0) wcount[warp][digit] = __popc(peers);
        __syncthreads();
#pragma unroll
        for (int w = 0; w < RS_WARPS; ++w) {
            woff[w][dgt] = run;
            run += wcount[w][dgt];
            wcount[w][dgt] = 0;
        }
        __syncthreads();
        if (live) {
            const unsigned pos = woff[warp][digit] + rank;
            keys_out[pos] = key;
            ids_out[pos] = id;
        }
    }
}

// offsets[k] = the first position of the sorted keys that is >= k, k = 0 .. sentinel + 1
__global__ void __launch_bounds__(TEX_THREADS) tex_segment_bounds_kernel(const unsigned* __restrict__ keys, long long n,
                                                                         unsigned sentinel, int* __restrict__ offsets)
{
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long k = (long long)blockIdx.x * TEX_THREADS + threadIdx.x; k <= (long long)sentinel + 1; k += stride) {
        long long lo = 0, hi = n;
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (__ldg(keys + mid) < (unsigned)k) lo = mid + 1;
            else hi = mid;
        }
        offsets[k] = (int)lo;
    }
}

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
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    tex_det_chunk_kernel<CT><<<chunk_blocks, TEX_THREADS, 0, stream>>>(a);
    return cudaGetLastError();
}

inline unsigned det_blocks(long long work, long long per_block)
{
    const long long b = (work + per_block - 1) / per_block;
    return (unsigned)(b < 1 ? 1 : (b < DET_GRID ? b : DET_GRID));
}

// sort passes: one per 8 bits of the largest key, the sentinel
inline int sort_passes(unsigned sentinel)
{
    int bits = 0;
    while (bits < 32 && (sentinel >> bits) != 0) ++bits;
    return (bits + 7) / 8;
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
                                                  const TexDetScratch& s, cudaStream_t stream, int* launches)
{
    // grad_indices is per lookup and has no atomics: the default kernel writes it
    if (!grad_texture || d.total == 0) return launch_texture_backward(texture, indices, grad_out, grad_texture, grad_indices, d,
                                                                      stream, launches);
    cudaError_t e;
    if (grad_indices && (e = launch_texture_backward(texture, indices, grad_out, nullptr, grad_indices, d, stream, launches)) !=
                            cudaSuccess)
        return e;
    if ((e = cudaMemsetAsync(s.counters, 0, 2 * sizeof(int), stream)) != cudaSuccess) return e;
    const unsigned sentinel = (unsigned)(d.TB * d.texels);
    const int tiles = (int)((d.total + RS_TILE - 1) / RS_TILE), passes = sort_passes(sentinel);
    for (int p = 0; p < passes; ++p) {
        const unsigned* kin = s.keys[(p + 1) & 1];
        const int* iin = s.ids[(p + 1) & 1];
        unsigned* kout = s.keys[p & 1];
        int* iout = s.ids[p & 1];
        if (p == 0) tex_sort_hist_kernel<true><<<tiles, RS_THREADS, 0, stream>>>(kin, indices, d, sentinel, 0, s.counts, tiles);
        else tex_sort_hist_kernel<false><<<tiles, RS_THREADS, 0, stream>>>(kin, indices, d, sentinel, 8 * p, s.counts, tiles);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        tex_sort_scan_kernel<<<RS_RADIX, RS_THREADS, 0, stream>>>(s.counts, s.digit_total, tiles);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        if (p == 0)
            tex_sort_scatter_kernel<true><<<tiles, RS_THREADS, 0, stream>>>(kin, iin, indices, d, sentinel, 0, s.counts,
                                                                             s.digit_total, tiles, kout, iout);
        else
            tex_sort_scatter_kernel<false><<<tiles, RS_THREADS, 0, stream>>>(kin, iin, indices, d, sentinel, 8 * p, s.counts,
                                                                              s.digit_total, tiles, kout, iout);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        *launches += 3;
    }
    const unsigned* keys = s.keys[(passes - 1) & 1];
    tex_segment_bounds_kernel<<<det_blocks((long long)sentinel + 2, TEX_THREADS), TEX_THREADS, 0, stream>>>(keys, d.total,
                                                                                                           sentinel, s.offsets);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    TexDetArgs a;
    a.indices = indices; a.grad_out = grad_out; a.ids = s.ids[(passes - 1) & 1]; a.offsets = s.offsets;
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
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    *launches += 4;
    return cudaSuccess;
}

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

// ---- mipmapped (trilinear) lookup (DESIGN.md §7.6) ------------------------------------------------------------------
//
// Level k of L is [TB, TH >> k, TW >> k, C]; levels 1 .. L-1 live in the caller's pyramid buffer (mip_offset).  Per
// lookup: lambda from the screen-space derivatives, l = floor(lambda), f = lambda - l, and
// out = (1-f) * bilinear_l + f * bilinear_{l+1}, with level l+1 not read when f == 0.  Level k >= 1 is read at
// (index + 0.5) * 2^-k - 0.5, level 0 at the index itself, so that f == 0 at l == 0 is mode bilinear bit for bit.

namespace {

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

// the bilinear lookup of channels c0 .. c0 + NV - 1 at taps t of a texture of width TW and C channels
template <int NV, bool VEC>
__device__ __forceinline__ void bilinear_rows(const float* tex, const Taps& t, int TW, int C, int c0, float v[NV])
{
    float t00[NV], t01[NV], t10[NV], t11[NV];
    load_row<NV, VEC>(tex + ((long long)t.r0 * TW + t.c0) * C + c0, t00);
    load_row<NV, VEC>(tex + ((long long)t.r0 * TW + t.c1) * C + c0, t01);
    load_row<NV, VEC>(tex + ((long long)t.r1 * TW + t.c0) * C + c0, t10);
    load_row<NV, VEC>(tex + ((long long)t.r1 * TW + t.c1) * C + c0, t11);
#pragma unroll
    for (int j = 0; j < NV; ++j) v[j] = bilinear(t00[j], t01[j], t10[j], t11[j], t.fr, t.fc);
}

// One lookup's two levels: taps and pointers of level l (0) and l + 1 (1; unused when f == 0)
struct Trilinear {
    Taps t0, t1;
    const float *p0, *p1;   // the lookup's texture at level l / l + 1
    int w0, w1;             // their widths
    Lod lod;
};

__device__ __forceinline__ Trilinear trilinear_of(float2 ix, float4 dv, const float* texture, const float* pyramid,
                                                  const TexDims& d, int L, long long g)
{
    Trilinear q;
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

// One thread per lookup, CT = C in 1..4 or 0 (any C, one channel at a time).  VEC: indices 8-, derivatives 16-byte
// aligned, out, texture and pyramid rows aligned for the vector loads and stores (the C = 3 store is staged as in
// texture_forward_kernel).
template <int CT, bool VEC>
__global__ void __launch_bounds__(TEX_THREADS) texture_trilinear_forward_kernel(const float* __restrict__ texture,
                                                                                const float* __restrict__ pyramid,
                                                                                const float* __restrict__ indices,
                                                                                const float* __restrict__ derivatives,
                                                                                float* __restrict__ out, TexDims d, int L)
{
    constexpr int NV = CT ? CT : 1;
    const int C = CT ? CT : d.C;
    __shared__ __align__(16) float stage[CT == 3 ? TEX_THREADS * 3 : 1];
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long base = (long long)blockIdx.x * TEX_THREADS + (threadIdx.x & ~31); base < d.total; base += stride) {
        const long long g = base + lane;
        Trilinear q;
        q.t0.valid = false;
        if (g < d.total) q = trilinear_of(load_index<VEC>(indices, g), load_derivatives<VEC>(derivatives, g), texture, pyramid, d,
                                          L, g);
        for (int c0 = 0; c0 < C; c0 += NV) {
            float v[NV];
#pragma unroll
            for (int j = 0; j < NV; ++j) v[j] = 0.f;
            if (q.t0.valid) {
                bilinear_rows<NV, VEC>(q.p0, q.t0, q.w0, C, c0, v);
                if (q.lod.f != 0.f) {
                    float u[NV];
                    bilinear_rows<NV, VEC>(q.p1, q.t1, q.w1, C, c0, u);
                    const float omf = __fsub_rn(1.0f, q.lod.f);
#pragma unroll
                    for (int j = 0; j < NV; ++j) v[j] = __fadd_rn(__fmul_rn(omf, v[j]), __fmul_rn(q.lod.f, u[j]));
                }
            }
            float* o = out + g * C + c0;
            if (VEC && CT == 4) {
                if (g < d.total) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1 % NV], v[2 % NV], v[3 % NV]);
            } else if (VEC && CT == 2) {
                if (g < d.total) *reinterpret_cast<float2*>(o) = make_float2(v[0], v[1 % NV]);
            } else if (VEC && CT == 3 && base + 32 <= d.total) {
                float* s = stage + (threadIdx.x & ~31) * 3;
#pragma unroll
                for (int j = 0; j < NV; ++j) s[lane * 3 + j] = v[j];
                __syncwarp();
                if (lane < 24) *reinterpret_cast<float4*>(out + base * 3 + lane * 4) = reinterpret_cast<const float4*>(s)[lane];
                __syncwarp();
            } else if (g < d.total) {
#pragma unroll
                for (int j = 0; j < NV; ++j) o[j] = v[j];
            }
        }
    }
}

// One thread per lookup, CT as in the forward kernel.  grad_indices per lookup, through both levels' fractions, each
// scaled by 2^-k.  The texel gradients of level 0 go to grad_texture, those of level k >= 1 to level_grad (the pyramid's
// layout), through the warp aggregation of texture_backward_kernel keyed on the packed texel index (level 0: its texel
// index; level k: TB * texels + the pyramid's texel index).
template <int CT, bool VEC>
__global__ void __launch_bounds__(TEX_THREADS) texture_trilinear_backward_kernel(
    const float* __restrict__ texture, const float* __restrict__ pyramid, const float* __restrict__ indices,
    const float* __restrict__ derivatives, const float* __restrict__ grad_out, float* __restrict__ grad_texture,
    float* __restrict__ level_grad, float* __restrict__ grad_indices, TexDims d, int L)
{
    constexpr int NV = CT ? CT : 1;
    const int C = CT ? CT : d.C;
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * TEX_THREADS;
    for (long long base = (long long)blockIdx.x * TEX_THREADS + (threadIdx.x & ~31); base < d.total; base += stride) {
        const long long g = base + lane;
        const bool live = g < d.total;
        Trilinear q;
        q.t0.valid = false;
        q.lod.l = 0; q.lod.f = 0.f;
        if (live) q = trilinear_of(load_index<VEC>(indices, g), load_derivatives<VEC>(derivatives, g), texture, pyramid, d, L, g);
        if (!q.t0.valid) {
            q.t0.r0 = q.t0.r1 = q.t0.c0 = q.t0.c1 = 0; q.t0.fr = q.t0.fc = 0.f; q.t0.base = 0;
            q.t1 = q.t0;
            q.lod.l = 0; q.lod.f = 0.f;
        }
        const bool both = q.t0.valid && q.lod.f != 0.f;
        const float omf = __fsub_rn(1.0f, q.lod.f);
        const float* gout = grad_out + g * C;
        float go[NV];
#pragma unroll
        for (int j = 0; j < NV; ++j) go[j] = 0.f;
        if (CT && q.t0.valid) load_row<NV, VEC>(gout, go);

        if (grad_indices && live) {
            float dr0 = 0.f, dc0 = 0.f, dr1 = 0.f, dc1 = 0.f;
            if (q.t0.valid) {
#pragma unroll
                for (int s = 0; s < 2; ++s) {
                    if (s == 1 && !both) break;
                    const Taps t = s ? q.t1 : q.t0;
                    const float* tex = s ? q.p1 : q.p0;
                    const int TW = s ? q.w1 : q.w0;
                    const float omr = __fsub_rn(1.0f, t.fr), omc = __fsub_rn(1.0f, t.fc);
                    float dr = 0.f, dc = 0.f;
                    for (int c0 = 0; c0 < C; c0 += NV) {
                        float t00[NV], t01[NV], t10[NV], t11[NV];
                        load_row<NV, VEC>(tex + ((long long)t.r0 * TW + t.c0) * C + c0, t00);
                        load_row<NV, VEC>(tex + ((long long)t.r0 * TW + t.c1) * C + c0, t01);
                        load_row<NV, VEC>(tex + ((long long)t.r1 * TW + t.c0) * C + c0, t10);
                        load_row<NV, VEC>(tex + ((long long)t.r1 * TW + t.c1) * C + c0, t11);
                        if (!CT) go[0] = __ldg(gout + c0);
#pragma unroll
                        for (int j = 0; j < NV; ++j) {
                            dc += go[j] * ((t01[j] - t00[j]) * omr + (t11[j] - t10[j]) * t.fr);
                            dr += go[j] * ((t10[j] - t00[j]) * omc + (t11[j] - t01[j]) * t.fc);
                        }
                    }
                    if (s) { dr1 = dr; dc1 = dc; }
                    else { dr0 = dr; dc0 = dc; }
                }
            }
            // d index_k / d index = 2^-k
            const float s0 = __int_as_float((127 - q.lod.l) << 23), s1 = 0.5f * s0;
            float dr = dr0 * s0, dc = dc0 * s0;
            if (both) {
                dr = omf * dr + q.lod.f * (dr1 * s1);
                dc = omf * dc + q.lod.f * (dc1 * s1);
            }
            if (VEC) reinterpret_cast<float2*>(grad_indices)[g] = make_float2(dr, dc);
            else { grad_indices[2 * g] = dr; grad_indices[2 * g + 1] = dc; }
        }

        if (grad_texture) {
#pragma unroll 1
            for (int s = 0; s < 2; ++s) {   // warp-uniform: every lane takes part in agg_plan
                const int k = q.lod.l + s;
                const Taps t = s ? q.t1 : q.t0;
                const float a = s ? q.lod.f : (both ? omf : 1.0f);
                const bool level_on = s ? both : q.t0.valid;
                const float omr = __fsub_rn(1.0f, t.fr), omc = __fsub_rn(1.0f, t.fc);
                const int TW = s ? q.w1 : q.w0;
                const long long first = k == 0 ? 0ll : (long long)d.TB * d.texels + mip_offset(d, k);
                float* dst_level = k == 0 ? grad_texture : level_grad + mip_offset(d, k) * C;
                for (int corner = 0; corner < 4; ++corner) {   // (r0,c0), (r0,c1), (r1,c0), (r1,c1)
                    const int r = (corner & 2) ? t.r1 : t.r0, c = (corner & 1) ? t.c1 : t.c0;
                    const float w = __fmul_rn(__fmul_rn((corner & 1) ? t.fc : omc, (corner & 2) ? t.fr : omr), a);
                    const bool on = level_on && w != 0.f;
                    const long long texel = t.base + (long long)r * TW + c;
                    const Agg ag = agg_plan(on ? (unsigned long long)(first + texel) : (1ull << 63) | (unsigned)lane, lane);
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
        }
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

template <int CT>
cudaError_t trilinear_forward_ct(const float* texture, const float* pyramid, const float* indices, const float* derivatives,
                                 float* out, const TexDims& d, int L, cudaStream_t stream)
{
    const int row = CT == 2 || CT == 4 ? 4 * CT : 4;
    const int out_bytes = CT == 3 ? 16 : row;
    const bool vec = CT && aligned(indices, 8) && aligned(derivatives, 16) && aligned(out, out_bytes) &&
                     aligned(texture, row) && aligned(pyramid, row);
    const unsigned blocks = blocks_for(d.total);
    if constexpr (CT != 0) {   // any C has no vector path
        if (vec) {
            texture_trilinear_forward_kernel<CT, true><<<blocks, TEX_THREADS, 0, stream>>>(texture, pyramid, indices,
                                                                                          derivatives, out, d, L);
            return cudaGetLastError();
        }
    }
    texture_trilinear_forward_kernel<CT, false><<<blocks, TEX_THREADS, 0, stream>>>(texture, pyramid, indices, derivatives,
                                                                                       out, d, L);
    return cudaGetLastError();
}

template <int CT>
cudaError_t trilinear_backward_ct(const float* texture, const float* pyramid, const float* indices, const float* derivatives,
                                  const float* grad_out, float* grad_texture, float* level_grad, float* grad_indices,
                                  const TexDims& d, int L, cudaStream_t stream)
{
    const int row = CT == 2 || CT == 4 ? 4 * CT : 4;
    const bool vec = CT && aligned(indices, 8) && aligned(derivatives, 16) && aligned(grad_indices, 8) &&
                     aligned(grad_out, row) && aligned(texture, row) && aligned(pyramid, row) && aligned(grad_texture, row) &&
                     aligned(level_grad, row);
    const unsigned blocks = blocks_for(d.total);
    if constexpr (CT != 0) {
        if (vec) {
            texture_trilinear_backward_kernel<CT, true><<<blocks, TEX_THREADS, 0, stream>>>(
                texture, pyramid, indices, derivatives, grad_out, grad_texture, level_grad, grad_indices, d, L);
            return cudaGetLastError();
        }
    }
    texture_trilinear_backward_kernel<CT, false><<<blocks, TEX_THREADS, 0, stream>>>(
            texture, pyramid, indices, derivatives, grad_out, grad_texture, level_grad, grad_indices, d, L);
    return cudaGetLastError();
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

cudaError_t launch_texture_mip_build(const float* texture, float* pyramid, const TexDims& d, cudaStream_t stream,
                                     int* launches)
{
    const int L = mip_levels(d.TH, d.TW);
    for (int k = 1; k < L; ++k) {
        const long long n = (long long)d.TB * (d.texels >> (2 * k)) * d.C;
        mip_build_kernel<<<blocks_for(n), TEX_THREADS, 0, stream>>>(level_base(texture, (const float*)pyramid, d, k - 1),
                                                                    pyramid + mip_offset(d, k) * d.C, n, d.TH >> k,
                                                                    d.TW >> k, d.C);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        ++*launches;
    }
    return cudaSuccess;
}

cudaError_t launch_texture_trilinear_forward(const float* texture, const float* pyramid, const float* indices,
                                             const float* derivatives, float* out, const TexDims& d, cudaStream_t stream,
                                             int* launches)
{
    const int L = mip_levels(d.TH, d.TW);
    cudaError_t e;
    switch (d.C) {
        case 1: e = trilinear_forward_ct<1>(texture, pyramid, indices, derivatives, out, d, L, stream); break;
        case 2: e = trilinear_forward_ct<2>(texture, pyramid, indices, derivatives, out, d, L, stream); break;
        case 3: e = trilinear_forward_ct<3>(texture, pyramid, indices, derivatives, out, d, L, stream); break;
        case 4: e = trilinear_forward_ct<4>(texture, pyramid, indices, derivatives, out, d, L, stream); break;
        default: e = trilinear_forward_ct<0>(texture, pyramid, indices, derivatives, out, d, L, stream);
    }
    if (e == cudaSuccess) ++*launches;
    return e;
}

cudaError_t launch_texture_trilinear_backward(const float* texture, const float* pyramid, const float* indices,
                                              const float* derivatives, const float* grad_out, float* grad_texture,
                                              float* grad_indices, const TexDims& d, bool deterministic,
                                              const MipScratch& s, cudaStream_t stream, int* launches)
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
        switch (d.C) {
            case 1: e = trilinear_backward_ct<1>(texture, pyramid, indices, derivatives, grad_out, gt, s.level_grad, grad_indices, d, L, stream); break;
            case 2: e = trilinear_backward_ct<2>(texture, pyramid, indices, derivatives, grad_out, gt, s.level_grad, grad_indices, d, L, stream); break;
            case 3: e = trilinear_backward_ct<3>(texture, pyramid, indices, derivatives, grad_out, gt, s.level_grad, grad_indices, d, L, stream); break;
            case 4: e = trilinear_backward_ct<4>(texture, pyramid, indices, derivatives, grad_out, gt, s.level_grad, grad_indices, d, L, stream); break;
            default: e = trilinear_backward_ct<0>(texture, pyramid, indices, derivatives, grad_out, gt, s.level_grad, grad_indices, d, L, stream);
        }
        if (e != cudaSuccess) return e;
        ++*launches;
    }
    if (!grad_texture) return cudaSuccess;
    if (deterministic) {
        // level k's gradient, every texel written, by the §7.5 path over the lookups that read level k
        for (int k = 0; k < L; ++k) {
            mip_level_terms_kernel<<<blocks_for(d.total), TEX_THREADS, 0, stream>>>(indices, derivatives, grad_out, d, L, k,
                                                                                     s.indices, s.grad_out);
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
            ++*launches;
            TexDims dk = d;
            dk.TH = d.TH >> k; dk.TW = d.TW >> k; dk.texels = d.texels >> (2 * k);
            float* gk = k == 0 ? grad_texture : s.level_grad + mip_offset(d, k) * d.C;
            if ((e = launch_texture_backward_deterministic(nullptr, s.indices, s.grad_out, gk, nullptr, dk,
                                                           carve_texture_det_scratch(s.det, dk), stream, launches)) !=
                cudaSuccess)
                return e;
        }
    }
    if (L > 1) {
        mip_collapse_kernel<<<blocks_for((long long)d.TB * d.texels * d.C), TEX_THREADS, 0, stream>>>(grad_texture, s.level_grad,
                                                                                                      d, L);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        ++*launches;
    }
    return cudaSuccess;
}

}  // namespace dirt
