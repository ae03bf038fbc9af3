// derivatives.cu -- screen-space derivatives of G-buffer attributes (DESIGN.md §7.7).
//
// One thread per pixel.  A covered pixel evaluates its face's TriInterp planes where exact::gbuffer_at does and returns
// d a_c / dx and d a_c / dy of the perspective-correct interpolant of the face's vertex attributes; a background pixel
// returns zeros.  No atomics and no reductions: every output is one thread's arithmetic on its own inputs.
#include "common.cuh"

namespace dirt {

constexpr int DERIV_THREADS = 256;
#ifndef DIRT_DERIV_MAX_BLOCKS
#define DIRT_DERIV_MAX_BLOCKS 0x7fffffffll
#endif
constexpr long long DERIV_MAX_BLOCKS = DIRT_DERIV_MAX_BLOCKS;   // gridDim.x; the pixel loop strides past it

struct DerivArgs {
    const int32_t* face_ids;     // [B*H*W]
    const float* attributes;     // [B, V, C]
    float* out;                  // [B*H*W, 2, K]
    const TriInterp* itp;        // [B*F]
    Header* header;
    unsigned long long expect_tag;   // != 0: the records are promised to carry this tag
    long long total, HW;
    double inv_HW;
    int W, V, F, C, c0, K;
};

// the CT attributes of one vertex row from channel c0 on; VEC: one vector load
template <int CT, bool VEC>
__device__ __forceinline__ void load_attrs(const float* p, float v[CT])
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

// With b_k = q_k / S and a = a2 + b0 (a0 - a2) + b1 (a1 - a2):
//   d a / dx = (a0 - a2) * (q0A - b0 sA) / S + (a1 - a2) * (q1A - b1 sA) / S,
// which is (sum_k a_k q_kA - a sA) / S with sum_k b_k = 1 taken out, and the same with the B coefficients for y.
// CT = K in {1, 2, 4}: the row of 2K floats is stored as one float2 / float4 / two float4 (the launcher checks the
// alignment), VEC additionally loads the K attributes of a vertex as one vector; CT = 0: any K, scalar loops.
template <int CT, bool VEC>
__global__ void __launch_bounds__(DERIV_THREADS) derivatives_kernel(DerivArgs a)
{
    const long long stride = (long long)gridDim.x * DERIV_THREADS;
    // a workspace that does not hold these records: flag it (dirt_workspace_status) and return NaN everywhere rather
    // than gather vertex rows through ids that belong to other geometry
    const bool stale = a.expect_tag != 0 && a.header->tag != a.expect_tag;
    if (stale && blockIdx.x == 0 && threadIdx.x == 0) a.header->error = 1;
    const int K = CT ? CT : a.K;
    for (long long p = (long long)blockIdx.x * DERIV_THREADS + threadIdx.x; p < a.total; p += stride) {
        const int face = __ldg(a.face_ids + p);
        // p = b * HW + row * W + col without a 64-bit division: the double quotient is off by at most one
        long long b = (long long)__dmul_rn((double)p, a.inv_HW);
        long long rem = p - b * a.HW;
        if (rem < 0) { --b; rem += a.HW; } else if (rem >= a.HW) { ++b; rem -= a.HW; }
        const int row = (int)rem / a.W, col = (int)rem - row * a.W;
        float* o = a.out + p * 2 * K;
        float bx0 = 0.f, bx1 = 0.f, by0 = 0.f, by1 = 0.f;
        const float *r0 = nullptr, *r1 = nullptr, *r2 = nullptr;
        const bool covered = !stale && (unsigned)face < (unsigned)a.F;
        if (covered) {
            const TriInterp t = load_interp(a.itp + b * a.F + face);
            const float4 g = exact::gbuffer_at(t, col, row);   // (b0, b1, b2, 1 / S) as the G-buffer holds them
            bx0 = __fmul_rn(__fmaf_rn(-g.x, t.sA, t.q0A), g.w);
            bx1 = __fmul_rn(__fmaf_rn(-g.y, t.sA, t.q1A), g.w);
            by0 = __fmul_rn(__fmaf_rn(-g.x, t.sB, t.q0B), g.w);
            by1 = __fmul_rn(__fmaf_rn(-g.y, t.sB, t.q1B), g.w);
            const float* attr = a.attributes + (size_t)b * a.V * a.C + a.c0;
            r0 = attr + (size_t)t.v0 * a.C; r1 = attr + (size_t)t.v1 * a.C; r2 = attr + (size_t)t.v2 * a.C;
        }
        if constexpr (CT > 0) {
            float dx[CT], dy[CT];
#pragma unroll
            for (int j = 0; j < CT; ++j) dx[j] = dy[j] = stale ? __int_as_float(0x7fc00000) : 0.f;
            if (covered) {
                float a0[CT], a1[CT], a2[CT];
                load_attrs<CT, VEC>(r0, a0); load_attrs<CT, VEC>(r1, a1); load_attrs<CT, VEC>(r2, a2);
#pragma unroll
                for (int j = 0; j < CT; ++j) {
                    const float d0 = __fsub_rn(a0[j], a2[j]), d1 = __fsub_rn(a1[j], a2[j]);
                    dx[j] = __fmaf_rn(d0, bx0, __fmul_rn(d1, bx1));
                    dy[j] = __fmaf_rn(d0, by0, __fmul_rn(d1, by1));
                }
            }
            if (CT == 1) {
                *reinterpret_cast<float2*>(o) = make_float2(dx[0], dy[0]);
            } else if (CT == 2) {
                *reinterpret_cast<float4*>(o) = make_float4(dx[0], dx[1 % CT], dy[0], dy[1 % CT]);
            } else {
                reinterpret_cast<float4*>(o)[0] = make_float4(dx[0], dx[1 % CT], dx[2 % CT], dx[3 % CT]);
                reinterpret_cast<float4*>(o)[1] = make_float4(dy[0], dy[1 % CT], dy[2 % CT], dy[3 % CT]);
            }
        } else {
            for (int j = 0; j < K; ++j) {
                float dx = stale ? __int_as_float(0x7fc00000) : 0.f, dy = dx;
                if (covered) {
                    const float a2 = __ldg(r2 + j);
                    const float d0 = __fsub_rn(__ldg(r0 + j), a2), d1 = __fsub_rn(__ldg(r1 + j), a2);
                    dx = __fmaf_rn(d0, bx0, __fmul_rn(d1, bx1));
                    dy = __fmaf_rn(d0, by0, __fmul_rn(d1, by1));
                }
                o[j] = dx;
                o[K + j] = dy;
            }
        }
    }
}

cudaError_t launch_gbuffer_derivatives(const int32_t* face_ids, const float* attributes, float* out, const Workspace& ws,
                                       const Dims& d, int first_channel, int count, unsigned long long expect_tag,
                                       cudaStream_t stream)
{
    DerivArgs a;
    a.face_ids = face_ids; a.attributes = attributes; a.out = out; a.itp = ws.itp; a.header = ws.header;
    a.expect_tag = expect_tag;
    a.HW = (long long)d.H * d.W;
    a.total = (long long)d.B * a.HW;
    a.inv_HW = 1.0 / (double)a.HW;
    a.W = d.W; a.V = d.V; a.F = d.F; a.C = d.C; a.c0 = first_channel; a.K = count;
    if (a.total == 0) return cudaSuccess;
    const long long want = (a.total + DERIV_THREADS - 1) / DERIV_THREADS;
    const unsigned blocks = (unsigned)(want < DERIV_MAX_BLOCKS ? want : DERIV_MAX_BLOCKS);
    // vector attribute loads: every row's channel c0 is as aligned as the vector
    const uintptr_t first = (uintptr_t)(attributes + first_channel);
    const bool vec2 = first % 8 == 0 && d.C % 2 == 0, vec4 = first % 16 == 0 && d.C % 4 == 0;
    const bool out8 = (uintptr_t)out % 8 == 0, out16 = (uintptr_t)out % 16 == 0;
    if (count == 1 && out8)
        derivatives_kernel<1, false><<<blocks, DERIV_THREADS, 0, stream>>>(a);
    else if (count == 2 && out16 && vec2)
        derivatives_kernel<2, true><<<blocks, DERIV_THREADS, 0, stream>>>(a);
    else if (count == 2 && out16)
        derivatives_kernel<2, false><<<blocks, DERIV_THREADS, 0, stream>>>(a);
    else if (count == 4 && out16 && vec4)
        derivatives_kernel<4, true><<<blocks, DERIV_THREADS, 0, stream>>>(a);
    else if (count == 4 && out16)
        derivatives_kernel<4, false><<<blocks, DERIV_THREADS, 0, stream>>>(a);
    else
        derivatives_kernel<0, false><<<blocks, DERIV_THREADS, 0, stream>>>(a);
    return launched();
}

}  // namespace dirt
