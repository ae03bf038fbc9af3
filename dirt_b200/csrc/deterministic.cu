// deterministic.cu -- the RasteriseGrad pass with reproducible vertex gradients (dirt_rasterise_backward_deterministic,
// DESIGN.md §7.4).  Same inputs, flags, channel groups, per-pixel terms and dilation decisions as backward.cu, but no
// float atomics: every vertex gradient is one float64 sum in a fixed order, rounded once to fp32.
//
// Per channel group, in group order:
//  (1) record pass, one thread per pixel: the Scharr sums and the dilation of backward.cu's reference-shaped tile path
//      (grad_pixel.cuh), giving the pixel's dL/dx, dL/dy and a one-byte dilation code; grad_background as the default
//      path writes it; and the pixel box of every face, grown with integer atomicMin over the pixels that reference it
//      (as their own face for the colour terms, as the receiver of their position terms), one atomic per distinct face
//      per warp (MATCH.ANY).
//  (2) face gather: every face sweeps its box in raster order and sums, in float64, the colour terms of its own pixels and
//      the position terms of the pixels whose code points at it, each recomputed at its source pixel from the face's
//      record.  A box of up to DET_WARP_BOX pixels is swept by one warp, a larger one by one CTA; thread t takes the
//      box's pixels t, t + threads, ... and the lanes' sums meet in a fixed butterfly, so the sum is a function of the
//      box alone.  The per-face partials [B*F][3 corners][3 + C] are written by the first group and added to by the others.
// Then (3) the vertex -> face-corner adjacency of every item's face table (normals.cu's builder) and (4) one thread per
// output row sums the partials of the row's corners in ascending corner id k*F + f, over the items in item order when
// the geometry is shared, and rounds once.
#include "../../include/dirt_b200.h"
#include "common.cuh"
#include "grad_pixel.cuh"

namespace dirt {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int DET_THREADS = 256;
constexpr int DET_WARPS = DET_THREADS / 32;
constexpr long long DET_WARP_BOX = 2048;   // boxes of more pixels are swept by a whole CTA
constexpr unsigned DET_LARGE_CTAS = 1024;  // CTAs of the large-box pass (each takes whole faces)
#ifndef DIRT_DET_MAX_BLOCKS
#define DIRT_DET_MAX_BLOCKS (1ll << 20)
#endif
constexpr long long DET_MAX_BLOCKS = DIRT_DET_MAX_BLOCKS;

struct DetArgs {
    const float* vertices;
    const float* pixels;
    const float* grad_pixels;
    const int32_t* face_ids;
    const TriInterp* itp;
    float* grad_background;
    unsigned char* codes;     // this group's code plane [B*H*W]
    float2* rec;              // [B*H*W] dL/dx, dL/dy
    uint4* boxes;             // [B*F] {min col, min row, ~max col, ~max row}; all ones = empty
    double* partial;          // [B*F][3][NP]
    int* large;               // [B*F] faces whose box the CTA pass sweeps
    int* large_count;
    Header* header;
    unsigned long long expect_tag;
    int B, H, W, V, F, cs, c0, NP, flags;
};

__device__ __forceinline__ long long grid_blocks_stride() { return (long long)gridDim.x * DET_THREADS; }

// Grows the boxes of the faces `key` (global face index, -1: none) over the pixels of the warp that name them: one
// leader per distinct key reduces the coordinates of its peers and issues the four atomics.
__device__ __forceinline__ void grow_boxes(uint4* __restrict__ boxes, int key, int col, int row)
{
    const int lane = threadIdx.x & 31;
    const unsigned peers = __match_any_sync(FULL, key);
    unsigned leaders = __ballot_sync(FULL, key >= 0 && lane == __ffs(peers) - 1);
    while (leaders) {
        const int l = __ffs(leaders) - 1;
        leaders &= leaders - 1;
        const bool mine = (peers >> l) & 1u;
        const unsigned c0 = __reduce_min_sync(FULL, mine ? (unsigned)col : ~0u);
        const unsigned r0 = __reduce_min_sync(FULL, mine ? (unsigned)row : ~0u);
        const unsigned c1 = __reduce_min_sync(FULL, mine ? ~(unsigned)col : ~0u);
        const unsigned r1 = __reduce_min_sync(FULL, mine ? ~(unsigned)row : ~0u);
        if (lane == l) {
            unsigned* bx = reinterpret_cast<unsigned*>(boxes + key);
            atomicMin(bx, c0); atomicMin(bx + 1, r0); atomicMin(bx + 2, c1); atomicMin(bx + 3, r1);
        }
    }
}

// (1) one thread per pixel; a warp takes 32 consecutive pixels (the loop is warp-uniform)
template <int N0>
__global__ void __launch_bounds__(DET_THREADS) det_record_kernel(DetArgs a)
{
    const long long HW = (long long)a.H * a.W, total = (long long)a.B * HW;
    const bool want_pos = !(a.flags & BWD_SKIP_POSITION), want_col = !(a.flags & BWD_SKIP_COLOUR);
    const int lane = threadIdx.x & 31;
    if (a.expect_tag != 0 && blockIdx.x == 0 && threadIdx.x == 0 && a.header->tag != a.expect_tag) a.header->error = 1;
    const float inf = __int_as_float(0x7f800000);
    for (long long p0 = (long long)blockIdx.x * DET_THREADS + (threadIdx.x & ~31); p0 < total; p0 += grid_blocks_stride()) {
        const long long p = p0 + lane;
        int key_col = -1, key_pos = -1, col = 0, row = 0;
        if (p < total) {
            const int b = (int)(p / HW), pix = (int)(p - b * HW);
            row = pix / a.W;
            col = pix - row * a.W;
            const int32_t* ids = a.face_ids + (size_t)b * HW;
            const TriInterp* itp_b = a.itp + (size_t)b * a.F;
            const int f_own = ids[pix];
            if (want_col) {
                // grad_background: grad_pixels where uncovered, 0 elsewhere
                for (int ch = 0; ch < N0; ++ch)
                    a.grad_background[p * a.cs + a.c0 + ch] = f_own < 0 ? __ldg(&a.grad_pixels[p * a.cs + a.c0 + ch]) : 0.f;
                key_col = f_own >= 0 ? b * a.F + f_own : -1;
            }
            int code = DIL_NONE;
            float2 r = make_float2(0.f, 0.f);
            if (want_pos) {
                TriInterp t_own;
                float4 g_own = make_float4(-1.f, -1.f, -1.f, inf);
                if (f_own >= 0) {
                    t_own = load_interp(itp_b + f_own);
                    g_own = exact::gbuffer_at(t_own, col, row);
                }
                const Frame d{a.B, a.H, a.W};
                float sx[3], sy[3];
                scharr_global<N0>(a.pixels, b, row, col, d, a.cs, a.c0, sx, sy);
                int f = f_own;
                float4 g = g_own;
                TriInterp tf = t_own;
                const bool interior = col > 0 && row > 0 && col < a.W - 1 && row < a.H - 1;
                int c = DIL_OWN;
                if (interior) dilate_generic(ids, itp_b, d, col, row, sx, sy, f_own, t_own, g_own, f, g, tf, c);
                if (f >= 0) {
                    float dLdx = 0.f, dLdy = 0.f;
                    for (int ch = 0; ch < N0; ++ch) {
                        const float gp = __ldg(&a.grad_pixels[p * a.cs + a.c0 + ch]);
                        dLdx += gp * sx[ch];
                        dLdy += gp * sy[ch];
                    }
                    code = c;
                    r = make_float2(dLdx, dLdy);
                    key_pos = b * a.F + f;
                }
            }
            a.codes[p] = (unsigned char)code;
            a.rec[p] = r;
        }
        grow_boxes(a.boxes, key_col, col, row);
        grow_boxes(a.boxes, key_pos != key_col ? key_pos : -1, col, row);
    }
}

// The sums of one face over the pixels t, t + nthreads, ... of its box (t = this thread's index among nthreads).
// s[0..8]: position terms (x, y, w of corners 0..2), s[9 + N0*k + ch]: colour terms of corner k, channel ch of the group.
template <int N0>
struct FaceSums {
    double s[9 + 3 * N0];
};

template <int N0>
__device__ __forceinline__ void sweep_face(const DetArgs& a, int gf, const uint4 box, int t, int nthreads, FaceSums<N0>& acc)
{
    const bool want_pos = !(a.flags & BWD_SKIP_POSITION), want_col = !(a.flags & BWD_SKIP_COLOUR);
    const int b = gf / a.F, f = gf - b * a.F;
    const TriInterp tr = load_interp(a.itp + gf);
    const int vid[3] = {tr.v0, tr.v1, tr.v2};
    float2 xy[3];
    const float* verts = a.vertices + (size_t)b * a.V * 4;
#pragma unroll
    for (int k = 0; k < 3; ++k) xy[k] = __ldg(reinterpret_cast<const float2*>(verts + (size_t)vid[k] * 4));
#pragma unroll
    for (int i = 0; i < 9 + 3 * N0; ++i) acc.s[i] = 0.0;
    const int x0 = (int)box.x, y0 = (int)box.y, bw = (int)~box.z - x0 + 1, bh = (int)~box.w - y0 + 1;
    const long long area = (long long)bw * bh;
    const size_t img = (size_t)b * a.H * a.W;
    for (long long i = t; i < area; i += nthreads) {
        const int dr = (int)(i / bw), col = x0 + (int)(i - (long long)dr * bw), row = y0 + dr;
        const size_t p = img + (size_t)row * a.W + col;
        const int own = a.face_ids[p];
        if (want_col && own == f) {
            const float4 g = exact::gbuffer_at(tr, col, row);
            const float bary[3] = {g.x, g.y, g.z};
#pragma unroll
            for (int ch = 0; ch < N0; ++ch) {
                const float gp = __ldg(&a.grad_pixels[p * a.cs + a.c0 + ch]);
#pragma unroll
                for (int k = 0; k < 3; ++k) acc.s[9 + N0 * k + ch] += (double)(gp * bary[k]);
            }
        }
        if (!want_pos) continue;
        const int code = a.codes[p], which = code & 3;
        if (which == DIL_NONE) continue;
        int nc = col, nr = row, fq = own;
        if (which != DIL_OWN) {
            // the neighbour the record pass chose: its step, dithered by (col+row)%2, reversed for the second attempt
            int dx = (code & DIL_ALONG_ROW) ? 1 : 0, dy = 1 - dx;
            if ((col + row) & 1) { dx = -dx; dy = -dy; }
            if (which == DIL_SECOND) { dx = -dx; dy = -dy; }
            nc = col + dx;
            nr = row - dy;
            fq = a.face_ids[img + (size_t)nr * a.W + nc];
        }
        if (fq != f) continue;
        // the position terms of backward.cu's reference-shaped path, at the fragment's source pixel
        const float4 g = exact::gbuffer_at(tr, nc, nr);
        const float2 r = a.rec[p];
        const float bary[3] = {g.x, g.y, g.z};
        float clip_x = 0.f, clip_y = 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            clip_x += bary[k] * xy[k].x;
            clip_y += bary[k] * xy[k].y;
        }
        const float inv_w = 1.f / g.w;
        const float dxv_dxc = 0.5f * (float)a.W * inv_w, dyv_dyc = 0.5f * (float)a.H * inv_w;
        const float dxv_dwc = -dxv_dxc * clip_x * inv_w, dyv_dwc = -dyv_dyc * clip_y * inv_w;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float ax = r.x * bary[k], ay = r.y * bary[k];
            acc.s[3 * k + 0] += (double)(ax * dxv_dxc);
            acc.s[3 * k + 1] += (double)(ay * dyv_dyc);
            acc.s[3 * k + 2] += (double)(ax * dxv_dwc + ay * dyv_dwc);
        }
    }
}

template <int N0>
__device__ __forceinline__ void warp_butterfly(FaceSums<N0>& acc)
{
#pragma unroll
    for (int i = 0; i < 9 + 3 * N0; ++i)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc.s[i] = __dadd_rn(acc.s[i], __shfl_xor_sync(FULL, acc.s[i], o));
}

// the first group writes the face's partials (the buffer starts zeroed for faces no group visits), later ones add
template <int N0>
__device__ __forceinline__ void store_partials(const DetArgs& a, int gf, const FaceSums<N0>& acc)
{
    double* q = a.partial + (size_t)gf * 3 * a.NP;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        q[k * a.NP + 0] = __dadd_rn(q[k * a.NP + 0], acc.s[3 * k + 0]);
        q[k * a.NP + 1] = __dadd_rn(q[k * a.NP + 1], acc.s[3 * k + 1]);
        q[k * a.NP + 2] = __dadd_rn(q[k * a.NP + 2], acc.s[3 * k + 2]);
#pragma unroll
        for (int ch = 0; ch < N0; ++ch) q[k * a.NP + 3 + a.c0 + ch] = acc.s[9 + N0 * k + ch];
    }
}

// (2a) one warp per face (warp-uniform loop over the B*F faces); larger boxes are listed for the CTA pass
template <int N0>
__global__ void __launch_bounds__(DET_THREADS) det_face_warp_kernel(DetArgs a)
{
    const int lane = threadIdx.x & 31;
    const long long faces = (long long)a.B * a.F;
    for (long long gf = (long long)blockIdx.x * DET_WARPS + (threadIdx.x >> 5); gf < faces; gf += (long long)gridDim.x * DET_WARPS) {
        const uint4 box = a.boxes[gf];
        if (box.x == ~0u) continue;
        const long long area = (long long)((int)~box.z - (int)box.x + 1) * ((int)~box.w - (int)box.y + 1);
        if (area > DET_WARP_BOX) {
            if (lane == 0) a.large[atomicAdd(a.large_count, 1)] = (int)gf;
            continue;
        }
        FaceSums<N0> acc;
        sweep_face<N0>(a, (int)gf, box, lane, 32, acc);
        warp_butterfly<N0>(acc);
        if (lane == 0) store_partials<N0>(a, (int)gf, acc);
    }
}

// (2b) one CTA per listed face; which CTA takes a face does not matter, the sum depends on the box alone
template <int N0>
__global__ void __launch_bounds__(DET_THREADS) det_face_cta_kernel(DetArgs a)
{
    constexpr int NS = 9 + 3 * N0;
    __shared__ double part[DET_WARPS][NS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = *a.large_count;
    for (int j = blockIdx.x; j < n; j += gridDim.x) {
        const int gf = a.large[j];
        FaceSums<N0> acc;
        sweep_face<N0>(a, gf, a.boxes[gf], threadIdx.x, DET_THREADS, acc);
        warp_butterfly<N0>(acc);
        if (lane == 0)
#pragma unroll
            for (int i = 0; i < NS; ++i) part[warp][i] = acc.s[i];
        __syncthreads();
        if (threadIdx.x == 0) {
#pragma unroll
            for (int i = 0; i < NS; ++i) {
                double s = part[0][i];
                for (int w = 1; w < DET_WARPS; ++w) s = __dadd_rn(s, part[w][i]);
                acc.s[i] = s;
            }
            store_partials<N0>(a, gf, acc);
        }
        __syncthreads();
    }
}

// (4) one thread per output row: grad_vertices [rows, 4] (column 2 is 0) and grad_vertex_colors [rows, C]
__global__ void __launch_bounds__(DET_THREADS) det_vertex_kernel(const int* __restrict__ offsets, const int* __restrict__ inc,
                                                                 const double* __restrict__ partial, float* __restrict__ gv,
                                                                 float* __restrict__ gc, int B, int V, int F, int C, bool shared,
                                                                 Header* header, unsigned long long expect_tag)
{
    const int NP = 3 + C;
    const long long rows = shared ? (long long)V : (long long)B * V;
    for (long long t = (long long)blockIdx.x * DET_THREADS + threadIdx.x; t < rows; t += grid_blocks_stride()) {
        const int b_first = shared ? 0 : (int)(t / V), b_end = shared ? B : b_first + 1;
        const int v = (int)(t - (shared ? 0 : (long long)b_first * V));
        for (int j = 0; j < NP; ++j) {
            double s = 0.0;
            for (int b = b_first; b < b_end; ++b) {
                const long long r = (long long)b * V + v;
                const int lo = __ldg(offsets + r), hi = __ldg(offsets + r + 1);
                for (int q = lo; q < hi; ++q) {
                    const int local = __ldg(inc + q) - b * 3 * F, k = local / F, f = local - k * F;
                    s = __dadd_rn(s, __ldg(partial + ((size_t)((long long)b * F + f) * 3 + k) * NP + j));
                }
            }
            const float x = __double2float_rn(s);
            if (j < 3) gv[t * 4 + (j == 2 ? 3 : j)] = x;
            else gc[t * C + (j - 3)] = x;
        }
        gv[t * 4 + 2] = 0.f;
        if (t == 0 && expect_tag != 0 && header->tag != expect_tag) gv[0] = __int_as_float(0x7fc00000);
    }
}

inline unsigned det_blocks(long long n, long long per_block)
{
    const long long b = (n + per_block - 1) / per_block;
    return (unsigned)(b < 1 ? 1 : (b < DET_MAX_BLOCKS ? b : DET_MAX_BLOCKS));
}

}  // namespace

DetScratch carve_det_scratch(void* base, int B, int H, int W, int C, int V, int F)
{
    DetScratch s = {};
    char* p = static_cast<char*>(base);
    unsigned __int128 off = 0;
    auto take = [&](unsigned __int128 bytes) {
        char* q = p ? p + (size_t)off : nullptr;
        off += (bytes + 255) / 256 * 256;
        return q;
    };
    const unsigned __int128 px = (unsigned __int128)B * H * W, bf = (unsigned __int128)B * F, bv = (unsigned __int128)B * V;
    s.codes = reinterpret_cast<unsigned char*>(take(px * C));
    s.rec = reinterpret_cast<float2*>(take(px * sizeof(float2)));
    s.boxes = reinterpret_cast<uint4*>(take(bf * sizeof(uint4)));
    s.large = reinterpret_cast<int*>(take(bf * sizeof(int)));
    s.large_count = reinterpret_cast<int*>(take(sizeof(int)));
    s.partial = reinterpret_cast<double*>(take(bf * 3 * (3 + (unsigned __int128)C) * sizeof(double)));
    s.offsets = reinterpret_cast<int*>(take((bv + 1) * sizeof(int)));
    s.counts = reinterpret_cast<int*>(take(bv * sizeof(int)));
    s.inc = reinterpret_cast<int*>(take(bf * 3 * sizeof(int)));
    s.unsorted = reinterpret_cast<int*>(take(bf * 3 * sizeof(int)));
    s.bytes = off > (unsigned __int128)SIZE_MAX ? SIZE_MAX : (size_t)off;
    return s;
}

cudaError_t launch_backward_deterministic(const float* vertices, const int32_t* faces, const float* pixels,
                                          const float* grad_pixels, const int32_t* face_ids, float* grad_background,
                                          float* grad_vertices, float* grad_vertex_colors, const Workspace& ws, const Dims& d,
                                          const GroupSpec& groups, int flags, unsigned long long expect_tag,
                                          const DetScratch& s, cudaStream_t stream)
{
    cudaError_t e;
    const long long px = (long long)d.B * d.H * d.W, faces_n = (long long)d.B * d.F;
    const int NP = 3 + d.C;
    if ((e = cudaMemsetAsync(s.partial, 0, sizeof(double) * 3 * NP * (size_t)faces_n, stream)) != cudaSuccess) return e;
    DetArgs a = {};
    a.vertices = vertices; a.pixels = pixels; a.grad_pixels = grad_pixels; a.face_ids = face_ids; a.itp = ws.itp;
    a.grad_background = grad_background; a.rec = s.rec; a.boxes = s.boxes; a.partial = s.partial; a.large = s.large;
    a.large_count = s.large_count; a.header = ws.header; a.expect_tag = expect_tag;
    a.B = d.B; a.H = d.H; a.W = d.W; a.V = d.V; a.F = d.F; a.cs = d.C; a.NP = NP; a.flags = flags;
    const unsigned large_ctas = (unsigned)(faces_n < DET_LARGE_CTAS ? (faces_n > 0 ? faces_n : 1) : DET_LARGE_CTAS);
    int c0 = 0;
    for (int g = 0; g < groups.n; ++g) {
        a.c0 = c0;
        a.codes = s.codes + (size_t)g * px;
        if ((e = cudaMemsetAsync(s.boxes, 0xff, sizeof(uint4) * (size_t)faces_n, stream)) != cudaSuccess) return e;
        if ((e = cudaMemsetAsync(s.large_count, 0, sizeof(int), stream)) != cudaSuccess) return e;
        const bool three = groups.width[g] == 3;
        if (three) det_record_kernel<3><<<det_blocks(px, DET_THREADS), DET_THREADS, 0, stream>>>(a);
        else det_record_kernel<1><<<det_blocks(px, DET_THREADS), DET_THREADS, 0, stream>>>(a);
        if ((e = launched()) != cudaSuccess) return e;
        if (faces_n > 0) {
            if (three) det_face_warp_kernel<3><<<det_blocks(faces_n, DET_WARPS), DET_THREADS, 0, stream>>>(a);
            else det_face_warp_kernel<1><<<det_blocks(faces_n, DET_WARPS), DET_THREADS, 0, stream>>>(a);
            if ((e = launched()) != cudaSuccess) return e;
            if (three) det_face_cta_kernel<3><<<large_ctas, DET_THREADS, 0, stream>>>(a);
            else det_face_cta_kernel<1><<<large_ctas, DET_THREADS, 0, stream>>>(a);
            if ((e = launched()) != cudaSuccess) return e;
        }
        c0 += groups.width[g];
    }
    const bool shared = (flags & BWD_SHARED_GEOMETRY) != 0;
    const long long rows = shared ? (long long)d.V : (long long)d.B * d.V;
    if (rows == 0) return cudaSuccess;
    if ((e = launch_corner_adjacency(faces, 3ll * d.F, d.B, d.V, d.F, s.counts, s.offsets, s.unsorted, s.inc, stream)) != cudaSuccess)
        return e;
    det_vertex_kernel<<<det_blocks(rows, DET_THREADS), DET_THREADS, 0, stream>>>(s.offsets, s.inc, s.partial, grad_vertices,
                                                                                 grad_vertex_colors, d.B, d.V, d.F, d.C, shared,
                                                                                 ws.header, expect_tag);
    return launched();
}

}  // namespace dirt
