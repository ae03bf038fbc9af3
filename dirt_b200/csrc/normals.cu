// normals.cu -- the vertex normals of dirt_b200/lighting.py (dirt_normals_forward / dirt_normals_backward,
// DESIGN.md §7.3): per vertex, the normalised sum of the unit normals of the faces using it, or, for pre-split meshes,
// the unit normal of its last face.
//
// The faces [F, 3] are shared by the batch, so the vertex -> incidence adjacency is built once per call, as CSR, from the
// faces alone: offsets[V + 1] and the incidence ids i = k*F + f (corner k of face f) of each vertex in ascending order,
// the order in which the restatement's three index_add calls visit them.  Faces with an index outside [0, V) are left
// out.  The build counts the incidences per vertex (integer atomics), scans the counts, drops the ids into their rows
// (integer atomics, in no fixed order) and then puts each id at its rank within its row, so the rows do not depend on
// scheduling.
//
// Every other pass is one thread per (item, vertex) that gathers over its row and recomputes what it needs of each face
// (its unit normal, or its corner gradients) from the positions: no per-face buffer, and no float atomics.  A row longer
// than LONG_ROW is summed by the whole warp instead (lane-strided partial sums, then a butterfly), so that a high-valence
// vertex does not hold up its warp's other 31 lanes.  Either way each sum has one fixed order for given faces, and two
// calls give bit-identical results.
//
// The file also holds the vertex tangents (dirt_tangents_forward / _backward, DESIGN.md §7.14), which use the same
// adjacency, workspace and per-vertex passes.
#include <cub/block/block_scan.cuh>

#include "../../include/dirt_b200.h"
#include "common.cuh"

namespace dirt {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int SCAN_THREADS = 1024;
#ifndef DIRT_NORMALS_MAX_BLOCKS
#define DIRT_NORMALS_MAX_BLOCKS (1ll << 20)
#endif
constexpr long long MAX_BLOCKS = DIRT_NORMALS_MAX_BLOCKS;

__device__ __forceinline__ float3 ld3(const float* p) { return make_float3(__ldg(p), __ldg(p + 1), __ldg(p + 2)); }
__device__ __forceinline__ void st3(float* p, float3 a) { p[0] = a.x; p[1] = a.y; p[2] = a.z; }
__device__ __forceinline__ float3 add3(float3 a, float3 b)
{
    return make_float3(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z));
}
__device__ __forceinline__ float3 sub3(float3 a, float3 b)
{
    return make_float3(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z));
}
__device__ __forceinline__ float dot3(float3 a, float3 b)
{
    return __fmaf_rn(a.z, b.z, __fmaf_rn(a.y, b.y, __fmul_rn(a.x, b.x)));
}
// torch.linalg.cross: (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0)
__device__ __forceinline__ float3 cross3(float3 a, float3 b)
{
    return make_float3(__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)),
                       __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
                       __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
}

// Two float3 summed side by side: the (t_f, b_f) of a face, or a corner's position and uv gradients.
struct Frame {
    float3 t, b;
};
__device__ __forceinline__ Frame add3(Frame a, Frame b) { return Frame{add3(a.t, b.t), add3(a.b, b.b)}; }
__device__ __forceinline__ float3 zero_of(float3) { return make_float3(0.f, 0.f, 0.f); }
__device__ __forceinline__ Frame zero_of(Frame) { return Frame{zero_of(float3()), zero_of(float3())}; }
// one butterfly step: p += p of the lane o away
__device__ __forceinline__ void add_xor(float3& p, int o)
{
    p.x = __fadd_rn(p.x, __shfl_xor_sync(FULL, p.x, o));
    p.y = __fadd_rn(p.y, __shfl_xor_sync(FULL, p.y, o));
    p.z = __fadd_rn(p.z, __shfl_xor_sync(FULL, p.z, o));
}
__device__ __forceinline__ void add_xor(Frame& p, int o)
{
    add_xor(p.t, o);
    add_xor(p.b, o);
}
__device__ __forceinline__ float3 scale3(float3 a, float k)
{
    return make_float3(__fmul_rn(a.x, k), __fmul_rn(a.y, k), __fmul_rn(a.z, k));
}

// x / (|x| + 1e-12)
__device__ __forceinline__ float3 normalise(float3 x)
{
    const float d = __fadd_rn(__fsqrt_rn(dot3(x, x)), 1.e-12f);
    return make_float3(__fdiv_rn(x.x, d), __fdiv_rn(x.y, d), __fdiv_rn(x.z, d));
}

// The gradient torch autograd gives `normalise` at x for the output gradient g: g / d through the numerator, and
// -(g . x) / d^2 through d = |x| + 1e-12 on to x, except through the norm of a zero vector.
__device__ __forceinline__ float3 normalise_grad(float3 x, float3 g)
{
    const float nr = __fsqrt_rn(dot3(x, x)), d = __fadd_rn(nr, 1.e-12f);
    const float gd = -__fdiv_rn(dot3(g, x), __fmul_rn(d, d));
    const float k = nr == 0.f ? 0.f : __fdiv_rn(gd, nr);
    return make_float3(__fmaf_rn(x.x, k, __fdiv_rn(g.x, d)), __fmaf_rn(x.y, k, __fdiv_rn(g.y, d)),
                       __fmaf_rn(x.z, k, __fdiv_rn(g.z, d)));
}

__device__ __forceinline__ bool load_face(const int* __restrict__ faces, long long f, int V, int v[3])
{
#pragma unroll
    for (int k = 0; k < 3; ++k) v[k] = __ldg(faces + 3 * f + k);
    return v[0] >= 0 && v[0] < V && v[1] >= 0 && v[1] < V && v[2] >= 0 && v[2] < V;
}

// The positions of the corners of face f of item b, and its edges from corner 0.
struct Corners {
    int v[3];
    float3 e1, e2;
};

__device__ __forceinline__ Corners corners(const NormalsArgs& a, long long b, int f)
{
    Corners c;
    load_face(a.faces, f, a.V, c.v);
    const float* base = a.vertices + b * a.V * a.stride;
    const float3 p0 = ld3(base + c.v[0] * a.stride);
    c.e1 = sub3(ld3(base + c.v[1] * a.stride), p0);
    c.e2 = sub3(ld3(base + c.v[2] * a.stride), p0);
    return c;
}

// ---- the adjacency ----------------------------------------------------------------------------------------------------

// The adjacency builder serves `items` face tables of F faces each, `face_stride` ints apart (0: one table shared by the
// batch).  Row b*V + v holds the incidences of vertex v in table b, as ids b*3F + k*F + f.

__global__ void __launch_bounds__(NORMALS_THREADS) count_kernel(const int* __restrict__ faces, long long face_stride, int items,
                                                                int F, int V, int* __restrict__ counts)
{
    const long long n = (long long)items * F;
    for (long long t = (long long)blockIdx.x * NORMALS_THREADS + threadIdx.x; t < n; t += (long long)gridDim.x * NORMALS_THREADS) {
        const long long b = t / F, f = t - b * F;
        int v[3];
        if (!load_face(faces + b * face_stride, f, V, v)) continue;
#pragma unroll
        for (int k = 0; k < 3; ++k) atomicAdd(counts + b * V + v[k], 1);
    }
}

// offsets[r] = sum of counts[0 .. r), for r in [0, n]: one CTA, each thread scanning a contiguous chunk
__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(const int* __restrict__ counts, long long n, int* __restrict__ offsets)
{
    using Scan = cub::BlockScan<int, SCAN_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const long long chunk = (n + SCAN_THREADS - 1) / SCAN_THREADS;
    const long long lo = threadIdx.x * chunk, hi = lo + chunk < n ? lo + chunk : n;
    int sum = 0;
    for (long long v = lo; v < hi; ++v) sum += counts[v];
    int run, total;
    Scan(tmp).ExclusiveSum(sum, run, total);
    for (long long v = lo; v < hi; ++v) {
        offsets[v] = run;
        run += counts[v];
    }
    if (threadIdx.x == 0) offsets[n] = total;
}

// Drops every incidence id into its vertex's row, at a place the atomics choose; counts[r] runs back down to 0.
__global__ void __launch_bounds__(NORMALS_THREADS) fill_kernel(const int* __restrict__ faces, long long face_stride, int items,
                                                               int F, int V, const int* __restrict__ offsets,
                                                               int* __restrict__ counts, int* __restrict__ unsorted)
{
    const long long n = (long long)items * F;
    for (long long t = (long long)blockIdx.x * NORMALS_THREADS + threadIdx.x; t < n; t += (long long)gridDim.x * NORMALS_THREADS) {
        const long long b = t / F, f = t - b * F;
        int v[3];
        if (!load_face(faces + b * face_stride, f, V, v)) continue;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const long long r = b * V + v[k];
            unsorted[offsets[r] + atomicSub(counts + r, 1) - 1] = (int)(b * 3 * F + k * F + f);
        }
    }
}

// Moves every id to its rank among the ids of its row: the rows in ascending order.
__global__ void __launch_bounds__(NORMALS_THREADS) rank_kernel(const int* __restrict__ faces, long long face_stride, int items,
                                                               int F, const int* __restrict__ offsets,
                                                               const int* __restrict__ unsorted, int* __restrict__ inc,
                                                               int V)
{
    const long long n = offsets[(long long)items * V];
    for (long long p = (long long)blockIdx.x * NORMALS_THREADS + threadIdx.x; p < n; p += (long long)gridDim.x * NORMALS_THREADS) {
        const int i = unsorted[p], b = i / (3 * F), local = i - b * 3 * F, k = local / F;
        const long long r = (long long)b * V + __ldg(faces + b * face_stride + 3ll * (local - k * F) + k);
        const int lo = offsets[r], hi = offsets[r + 1];
        int rank = 0;
        for (int j = lo; j < hi; ++j) rank += unsorted[j] < i;
        inc[lo + rank] = i;
    }
}

// ---- the per-vertex passes --------------------------------------------------------------------------------------------

// The sum over the row [lo, hi) of item b of term(b, i) for its incidence ids i.  Rows of up to LONG_ROW ids are summed by
// their own lane in row order; longer rows by the whole warp, one after another, each lane summing every 32nd id and the
// warp adding the lanes' sums as a butterfly.  Warp-collective: every lane calls it, inactive ones with an empty row.
// The terms are float3 (normals) or Frame (tangent frames and their gradients), summed component by component.
template <class Term>
__device__ __forceinline__ auto row_sum(const int* __restrict__ inc, int lo, int hi, long long b, const Term& term)
    -> decltype(term(b, 0))
{
    using T = decltype(term(b, 0));
    const int lane = threadIdx.x & 31;
    T s = zero_of(T());
    const bool long_row = hi - lo > NORMALS_LONG_ROW;
    if (!long_row)
        for (int j = lo; j < hi; ++j) s = add3(s, term(b, __ldg(inc + j)));
    unsigned pending = __ballot_sync(FULL, long_row);
    while (pending) {
        const int src = __ffs(pending) - 1;
        pending &= pending - 1;
        const int l = __shfl_sync(FULL, lo, src), h = __shfl_sync(FULL, hi, src);
        const long long bb = __shfl_sync(FULL, b, src);
        T p = zero_of(T());
        for (int j = l + lane; j < h; j += 32) p = add3(p, term(bb, __ldg(inc + j)));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) add_xor(p, o);
        if (lane == src) s = p;
    }
    return s;
}

// u_f of the face of incidence i
struct FaceUnit {
    const NormalsArgs& a;
    __device__ __forceinline__ float3 operator()(long long b, int i) const
    {
        const int f = i % a.F;
        const Corners c = corners(a, b, f);
        return normalise(cross3(c.e1, c.e2));
    }
};

// The gradient of corner k of the face of incidence i = k*F + f.  g_u of the face is the sum over its corners k' of
// the gradient of the vertex they feed: gs (average), or, pre-split, grad_normals where the incidence k'*F + f is the
// last of its vertex's row.
template <int MODE>
struct CornerGrad {
    const NormalsArgs& a;
    __device__ __forceinline__ float3 operator()(long long b, int i) const
    {
        const int k = i / a.F, f = i - k * a.F;
        const Corners c = corners(a, b, f);
        float3 gu = make_float3(0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const long long row = b * a.V + c.v[j];
            if (MODE == DIRT_NORMALS_AVERAGE) gu = add3(gu, ld3(a.gs + 3 * row));
            else if (__ldg(a.inc + __ldg(a.offsets + c.v[j] + 1) - 1) == j * a.F + f)
                gu = add3(gu, ld3(a.grad + 3 * row));
        }
        const float3 gn = normalise_grad(cross3(c.e1, c.e2), gu);
        const float3 g1 = cross3(c.e2, gn), g2 = cross3(gn, c.e1);   // d/d e1, d/d e2
        if (k == 1) return g1;
        if (k == 2) return g2;
        return make_float3(-__fadd_rn(g1.x, g2.x), -__fadd_rn(g1.y, g2.y), -__fadd_rn(g1.z, g2.z));
    }
};

// The threads of a warp take consecutive (item, vertex) rows t = b*V + v; the loop is warp-uniform.
#define FOR_EACH_ROW(a)                                                                                                \
    for (long long t0 = (long long)blockIdx.x * NORMALS_THREADS + (threadIdx.x & ~31); t0 < (a).total;               \
         t0 += (long long)gridDim.x * NORMALS_THREADS)

struct Row {
    long long t, b;
    int lo, hi;
    bool active;
};

__device__ __forceinline__ Row row_of(const NormalsArgs& a, long long t0)
{
    Row r;
    r.t = t0 + (threadIdx.x & 31);
    r.active = r.t < a.total;
    r.b = r.active ? r.t / a.V : 0;
    const long long v = r.t - r.b * a.V;
    r.lo = r.hi = 0;
    if (r.active) {
        r.lo = __ldg(a.offsets + v);
        r.hi = __ldg(a.offsets + v + 1);
    }
    return r;
}

template <int MODE>
__global__ void __launch_bounds__(NORMALS_THREADS) normals_forward_kernel(NormalsArgs a)
{
    FOR_EACH_ROW(a) {
        const Row r = row_of(a, t0);
        float3 n;
        if (MODE == DIRT_NORMALS_AVERAGE) {
            n = normalise(row_sum(a.inc, r.lo, r.hi, r.b, FaceUnit{a}));
        } else {
            n = r.hi > r.lo ? FaceUnit{a}(r.b, __ldg(a.inc + r.hi - 1)) : make_float3(0.f, 0.f, 0.f);
        }
        if (r.active) st3(a.out + 3 * r.t, n);
    }
}

// average mode: gs = the gradient of the vertex's sum of face normals
__global__ void __launch_bounds__(NORMALS_THREADS) normals_sum_grad_kernel(NormalsArgs a)
{
    FOR_EACH_ROW(a) {
        const Row r = row_of(a, t0);
        const float3 s = row_sum(a.inc, r.lo, r.hi, r.b, FaceUnit{a});
        if (r.active) st3(a.gs + 3 * r.t, normalise_grad(s, ld3(a.grad + 3 * r.t)));
    }
}

template <int MODE>
__global__ void __launch_bounds__(NORMALS_THREADS) normals_position_grad_kernel(NormalsArgs a)
{
    FOR_EACH_ROW(a) {
        const Row r = row_of(a, t0);
        const float3 g = row_sum(a.inc, r.lo, r.hi, r.b, CornerGrad<MODE>{a});
        if (r.active) st3(a.g_vertices + 3 * r.t, g);
    }
}

inline unsigned blocks_for(long long n)
{
    const long long b = (n + NORMALS_THREADS - 1) / NORMALS_THREADS;
    return (unsigned)(b < 1 ? 1 : (b < MAX_BLOCKS ? b : MAX_BLOCKS));
}

// ---- the vertex tangents (DESIGN.md §7.14) ------------------------------------------------------------------------------
//
// Face f with corners p0, p1, p2 and uvs (u_k, v_k): e1 = p1 - p0, e2 = p2 - p0, (du_k, dv_k) = uv_k - uv0,
// s = sign(du1 dv2 - du2 dv1), t_f = unit(s (e1 dv2 - e2 dv1)), b_f = unit(s (e2 du1 - e1 du2)).  The vertex passes sum
// t_f (and b_f) over the rows of the normals' adjacency, recomputing each face as the normals' passes do.

// A face's edges, its uv differences and the sign of its uv area.
struct UvFace {
    Corners c;
    float du1, dv1, du2, dv2, s;
};

__device__ __forceinline__ const float* uv_row(const TangentArgs& a, long long b, int v)
{
    return a.uvs + b * a.uv_item_stride + v * a.uv_stride;
}

__device__ __forceinline__ UvFace uv_face(const TangentArgs& a, long long b, int f)
{
    UvFace u;
    u.c = corners(a.m, b, f);
    const float* q0 = uv_row(a, b, u.c.v[0]);
    const float* q1 = uv_row(a, b, u.c.v[1]);
    const float* q2 = uv_row(a, b, u.c.v[2]);
    const float u0 = __ldg(q0), v0 = __ldg(q0 + 1);
    u.du1 = __fsub_rn(__ldg(q1), u0);
    u.dv1 = __fsub_rn(__ldg(q1 + 1), v0);
    u.du2 = __fsub_rn(__ldg(q2), u0);
    u.dv2 = __fsub_rn(__ldg(q2 + 1), v0);
    const float r = __fsub_rn(__fmul_rn(u.du1, u.dv2), __fmul_rn(u.du2, u.dv1));
    u.s = r > 0.f ? 1.f : (r < 0.f ? -1.f : 0.f);
    return u;
}

// s (e1 dv2 - e2 dv1): the face's unnormalised dp/du direction
__device__ __forceinline__ float3 face_u(const UvFace& u)
{
    const float3 e1 = u.c.e1, e2 = u.c.e2;
    return make_float3(__fmul_rn(u.s, __fsub_rn(__fmul_rn(e1.x, u.dv2), __fmul_rn(e2.x, u.dv1))),
                       __fmul_rn(u.s, __fsub_rn(__fmul_rn(e1.y, u.dv2), __fmul_rn(e2.y, u.dv1))),
                       __fmul_rn(u.s, __fsub_rn(__fmul_rn(e1.z, u.dv2), __fmul_rn(e2.z, u.dv1))));
}

// (t_f, b_f) of the face of incidence i
struct FaceFrame {
    const TangentArgs& a;
    __device__ __forceinline__ Frame operator()(long long b, int i) const
    {
        const UvFace u = uv_face(a, b, i % a.m.F);
        const float3 e1 = u.c.e1, e2 = u.c.e2;
        const float3 y = make_float3(__fmul_rn(u.s, __fsub_rn(__fmul_rn(e2.x, u.du1), __fmul_rn(e1.x, u.du2))),
                                     __fmul_rn(u.s, __fsub_rn(__fmul_rn(e2.y, u.du1), __fmul_rn(e1.y, u.du2))),
                                     __fmul_rn(u.s, __fsub_rn(__fmul_rn(e2.z, u.du1), __fmul_rn(e1.z, u.du2))));
        return Frame{normalise(face_u(u)), normalise(y)};
    }
};

// t_f alone (the backward's vertex pass)
struct FaceTangent {
    const TangentArgs& a;
    __device__ __forceinline__ float3 operator()(long long b, int i) const
    {
        return normalise(face_u(uv_face(a, b, i % a.m.F)));
    }
};

// The gradients of corner k of the face of incidence i = k*F + f: to its position (t) and to its v coordinate (b.y;
// b.x and b.z stay 0, as du reaches t_f only through the sign).  g_t of the face is the sum over its corners of the
// gradient of the vertex they feed.
struct TangentCornerGrad {
    const TangentArgs& a;
    __device__ __forceinline__ Frame operator()(long long b, int i) const
    {
        const int k = i / a.m.F, f = i - k * a.m.F;
        const UvFace u = uv_face(a, b, f);
        float3 gt = make_float3(0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 3; ++j) gt = add3(gt, ld3(a.gt + 3 * (b * a.m.V + u.c.v[j])));
        const float3 gy = scale3(normalise_grad(face_u(u), gt), u.s);   // to e1 dv2 - e2 dv1
        const float3 g1 = scale3(gy, u.dv2), g2 = scale3(gy, -u.dv1);   // d/d e1, d/d e2
        const float gdv2 = dot3(gy, u.c.e1), gdv1 = -dot3(gy, u.c.e2);
        Frame g = zero_of(Frame());
        if (k == 1) {
            g.t = g1;
            g.b.y = gdv1;
        } else if (k == 2) {
            g.t = g2;
            g.b.y = gdv2;
        } else {
            g.t = make_float3(-__fadd_rn(g1.x, g2.x), -__fadd_rn(g1.y, g2.y), -__fadd_rn(g1.z, g2.z));
            g.b.y = -__fadd_rn(gdv1, gdv2);
        }
        return g;
    }
};

// A row with no incidences (F = 0: there is no adjacency to read)
__device__ __forceinline__ Row tangent_row(const TangentArgs& a, long long t0)
{
    if (a.m.F) return row_of(a.m, t0);
    Row r;
    r.t = t0 + (threadIdx.x & 31);
    r.active = r.t < a.m.total;
    r.b = 0;
    r.lo = r.hi = 0;
    return r;
}

// n = unit(normal), x = t - (n . t) n: the vector T normalises
struct Gram {
    float3 n, x;
    float d;
};

__device__ __forceinline__ Gram gram(const TangentArgs& a, const Row& r, float3 t)
{
    Gram g;
    g.n = r.active ? normalise(ld3(a.normals + r.t * a.normal_stride)) : make_float3(0.f, 0.f, 0.f);
    g.d = dot3(g.n, t);
    g.x = sub3(t, scale3(g.n, g.d));
    return g;
}

__global__ void __launch_bounds__(NORMALS_THREADS) tangents_forward_kernel(TangentArgs a)
{
    FOR_EACH_ROW(a.m) {
        const Row r = tangent_row(a, t0);
        const Frame s = row_sum(a.m.inc, r.lo, r.hi, r.b, FaceFrame{a});
        const Gram g = gram(a, r, s.t);
        const float3 T = normalise(g.x);
        const float w = dot3(cross3(g.n, T), s.b) < 0.f ? -1.f : 1.f;
        if (r.active) {
            st3(a.out + 4 * r.t, T);
            a.out[4 * r.t + 3] = w;
        }
    }
}

// gt = the gradient of the vertex's sum of face tangents; grad_normals, which is local to the vertex
__global__ void __launch_bounds__(NORMALS_THREADS) tangents_vertex_grad_kernel(TangentArgs a)
{
    FOR_EACH_ROW(a.m) {
        const Row r = tangent_row(a, t0);
        const float3 t = row_sum(a.m.inc, r.lo, r.hi, r.b, FaceTangent{a});
        if (!r.active) continue;
        const Gram g = gram(a, r, t);
        const float3 gx = normalise_grad(g.x, ld3(a.grad + 4 * r.t));
        const float gxn = dot3(gx, g.n);
        // x = t - d n, d = n . t:  g_t = gx - (gx . n) n,  g_n = -d gx - (gx . n) t
        if (a.gt) st3(a.gt + 3 * r.t, sub3(gx, scale3(g.n, gxn)));
        if (a.g_normals) {
            const float3 gn = sub3(scale3(gx, -g.d), scale3(t, gxn));
            st3(a.g_normals + 3 * r.t, normalise_grad(ld3(a.normals + r.t * a.normal_stride), gn));
        }
    }
}

__global__ void __launch_bounds__(NORMALS_THREADS) tangents_corner_grad_kernel(TangentArgs a)
{
    FOR_EACH_ROW(a.m) {
        const Row r = tangent_row(a, t0);
        const Frame g = row_sum(a.m.inc, r.lo, r.hi, r.b, TangentCornerGrad{a});
        if (!r.active) continue;
        if (a.g_vertices) st3(a.g_vertices + 3 * r.t, g.t);
        if (a.g_uvs) {
            a.g_uvs[2 * r.t] = 0.f;
            a.g_uvs[2 * r.t + 1] = g.b.y;
        }
    }
}

}  // namespace

NormalsWorkspace carve_normals_workspace(void* base, int B, long long V, long long F)
{
    NormalsWorkspace w = {};
    char* p = static_cast<char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char* q = p ? p + off : nullptr;
        off += (bytes + 255) & ~size_t(255);
        return q;
    };
    w.offsets = reinterpret_cast<int*>(take(sizeof(int) * (size_t)(V + 1)));
    w.inc = reinterpret_cast<int*>(take(sizeof(int) * (size_t)(3 * F)));
    // the build's scratch (counts, unsorted ids) and the backward's per-vertex gradients share one region
    const size_t build = ((sizeof(int) * (size_t)V + 255) & ~size_t(255)) + sizeof(int) * (size_t)(3 * F);
    const size_t grads = sizeof(float) * 3 * (size_t)B * (size_t)V;
    char* scratch = take(build > grads ? build : grads);
    w.counts = reinterpret_cast<int*>(scratch);
    w.unsorted = scratch ? reinterpret_cast<int*>(scratch + ((sizeof(int) * (size_t)V + 255) & ~size_t(255))) : nullptr;
    w.gs = reinterpret_cast<float*>(scratch);
    w.bytes = off;
    return w;
}

cudaError_t launch_corner_adjacency(const int* faces, long long face_stride, int items, int V, int F, int* counts, int* offsets,
                                    int* unsorted, int* inc, cudaStream_t stream)
{
    cudaError_t e;
    const long long rows = (long long)items * V, corners = 3ll * items * F;
    if ((e = cudaMemsetAsync(counts, 0, sizeof(int) * (size_t)rows, stream)) != cudaSuccess) return e;
    count_kernel<<<blocks_for(corners / 3), NORMALS_THREADS, 0, stream>>>(faces, face_stride, items, F, V, counts);
    if ((e = launched()) != cudaSuccess) return e;
    scan_kernel<<<1, SCAN_THREADS, 0, stream>>>(counts, rows, offsets);
    if ((e = launched()) != cudaSuccess) return e;
    fill_kernel<<<blocks_for(corners / 3), NORMALS_THREADS, 0, stream>>>(faces, face_stride, items, F, V, offsets, counts, unsorted);
    if ((e = launched()) != cudaSuccess) return e;
    rank_kernel<<<blocks_for(corners), NORMALS_THREADS, 0, stream>>>(faces, face_stride, items, F, offsets, unsorted, inc, V);
    return launched();
}

cudaError_t launch_normals_forward(NormalsArgs a, const NormalsWorkspace& w, cudaStream_t stream)
{
    cudaError_t e;
    if (a.total == 0) return cudaSuccess;
    if (a.F == 0) return cudaMemsetAsync(a.out, 0, sizeof(float) * 3 * (size_t)a.total, stream);
    if ((e = launch_corner_adjacency(a.faces, 0, 1, a.V, a.F, w.counts, w.offsets, w.unsorted, w.inc, stream)) != cudaSuccess)
        return e;
    a.offsets = w.offsets;
    a.inc = w.inc;
    if (a.mode == DIRT_NORMALS_AVERAGE)
        normals_forward_kernel<DIRT_NORMALS_AVERAGE><<<blocks_for(a.total), NORMALS_THREADS, 0, stream>>>(a);
    else
        normals_forward_kernel<DIRT_NORMALS_PRE_SPLIT><<<blocks_for(a.total), NORMALS_THREADS, 0, stream>>>(a);
    return launched();
}

cudaError_t launch_normals_backward(NormalsArgs a, const NormalsWorkspace& w, cudaStream_t stream)
{
    cudaError_t e;
    if (a.total == 0) return cudaSuccess;
    if (a.F == 0) return cudaMemsetAsync(a.g_vertices, 0, sizeof(float) * 3 * (size_t)a.total, stream);
    a.offsets = w.offsets;
    a.inc = w.inc;
    a.gs = w.gs;
    if (a.mode == DIRT_NORMALS_AVERAGE) {
        normals_sum_grad_kernel<<<blocks_for(a.total), NORMALS_THREADS, 0, stream>>>(a);
        if ((e = launched()) != cudaSuccess) return e;
        normals_position_grad_kernel<DIRT_NORMALS_AVERAGE><<<blocks_for(a.total), NORMALS_THREADS, 0, stream>>>(a);
    } else {
        normals_position_grad_kernel<DIRT_NORMALS_PRE_SPLIT><<<blocks_for(a.total), NORMALS_THREADS, 0, stream>>>(a);
    }
    return launched();
}

cudaError_t launch_tangents_forward(TangentArgs a, const NormalsWorkspace& w, cudaStream_t stream)
{
    cudaError_t e;
    if (a.m.total == 0) return cudaSuccess;
    if (a.m.F > 0 &&
        (e = launch_corner_adjacency(a.m.faces, 0, 1, a.m.V, a.m.F, w.counts, w.offsets, w.unsorted, w.inc, stream)) != cudaSuccess)
        return e;
    a.m.offsets = w.offsets;
    a.m.inc = w.inc;
    tangents_forward_kernel<<<blocks_for(a.m.total), NORMALS_THREADS, 0, stream>>>(a);
    return launched();
}

cudaError_t launch_tangents_backward(TangentArgs a, const NormalsWorkspace& w, cudaStream_t stream)
{
    cudaError_t e;
    if (a.m.total == 0) return cudaSuccess;
    const size_t rows = (size_t)a.m.total;
    if (a.m.F == 0) {
        // every row is empty: T = 0 whatever the inputs, so no gradient reaches anything
        if (a.g_vertices && (e = cudaMemsetAsync(a.g_vertices, 0, sizeof(float) * 3 * rows, stream)) != cudaSuccess) return e;
        if (a.g_uvs && (e = cudaMemsetAsync(a.g_uvs, 0, sizeof(float) * 2 * rows, stream)) != cudaSuccess) return e;
        if (a.g_normals && (e = cudaMemsetAsync(a.g_normals, 0, sizeof(float) * 3 * rows, stream)) != cudaSuccess) return e;
        return cudaSuccess;
    }
    const bool corner = a.g_vertices || a.g_uvs;
    if (!corner && !a.g_normals) return cudaSuccess;
    a.m.offsets = w.offsets;
    a.m.inc = w.inc;
    a.gt = corner ? w.gs : nullptr;
    tangents_vertex_grad_kernel<<<blocks_for(a.m.total), NORMALS_THREADS, 0, stream>>>(a);
    if ((e = launched()) != cudaSuccess) return e;
    if (corner) {
        tangents_corner_grad_kernel<<<blocks_for(a.m.total), NORMALS_THREADS, 0, stream>>>(a);
        if ((e = launched()) != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace dirt
