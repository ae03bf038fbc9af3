// setup.cu -- triangle setup and per-tile binning.
//
// Replaces, for the sm_90a path, what the reference delegates to the OpenGL vertex pipeline
// (clip -> NDC -> viewport; csrc/rasterise_egl.cpp:362-380) and the vertex expansion kernel
// upload_vertices (csrc/rasterise_grad_egl.cu:12-34).
//
//   setup_kernel : one thread per (image, face): S1-S6 of the visibility specification ->
//                  TriCov + TriInterp + TriXY records, and -- in the same pass -- binning: the face is appended to the
//                  fixed-capacity bin of every tile its bounding box touches (faces spanning <= SMALL_TILE_LIMIT
//                  tiles; position = atomicAdd on the tile's count, overflow -> the image's overflow list) or to
//                  the per-image large list.  The order inside a bin is irrelevant: visibility is the minimum of
//                  (depth key, face index).  No scan, no second pass.
//                  A warp stages its 32 faces' records in shared memory and writes each record array with coalesced
//                  16-byte stores, and takes one atomicAdd per distinct tile of its faces' bounding boxes.
#include "common.cuh"

namespace dirt {

constexpr float GUARD_BAND = 8388608.0f;  // 2^23 sub-pixel units = 32768 px

// 128 threads x 4 blocks per SM (<= 128 registers: no spills; H100, DESIGN.md section 5)
#ifndef DIRT_SETUP_THREADS
#define DIRT_SETUP_THREADS 128
#endif
#ifndef DIRT_SETUP_MIN_BLOCKS
#define DIRT_SETUP_MIN_BLOCKS 4
#endif
#ifndef DIRT_SETUP_ABLATE
#define DIRT_SETUP_ABLATE 0   // timing builds only: 1 = no bin placement (no atomics, no bin stores), 2 = no shading record,
#endif                        // 3 = no coverage / interpolation / xy record stores (their values still computed), 4 = loads
                              // and the first culls only.  The forward call then skips the raster kernel (records undefined).

// Timing builds: a record store that DIRT_SETUP_ABLATE drops still feeds a value the compiler cannot discard
struct AblationSink {
    uint32_t v = 0;
    Header* h;
    __device__ explicit AblationSink(Header* header) : h(header) {}
    __device__ void take(uint4 u) { v ^= u.x ^ u.y ^ u.z ^ u.w; }
    __device__ ~AblationSink() { if (DIRT_SETUP_ABLATE != 0 && v == 0x9e3779b9u) h->pad = (int)v; }
};

// One warp's records on their way out.  A lane writes its own record (16-byte chunks, 64 or 32 bytes apart); the warp then
// stores each array as consecutive 16-byte chunks, 512 contiguous bytes per instruction.  Chunk c of the record of lane r
// sits at slot 4r + (c ^ ((r >> 1) & 3)) (64-byte records) or 2r + (c ^ ((r >> 2) & 1)) (32-byte ones): each 8-lane
// phase of either access touches 8 different 16-byte bank groups.
struct SetupStage {
    uint4 cov[128], itp[128], shade[128], xy[64];
};
__device__ __forceinline__ int slot64(int r, int c) { return 4 * r + (c ^ ((r >> 1) & 3)); }
__device__ __forceinline__ int slot32(int r, int c) { return 2 * r + (c ^ ((r >> 2) & 1)); }

constexpr int BIN_NONE = 0, BIN_SMALL = 1, BIN_LARGE = 2;

template <bool BIN>
__global__ void __launch_bounds__(DIRT_SETUP_THREADS, DIRT_SETUP_MIN_BLOCKS) setup_kernel(const float* __restrict__ vertices,
                                                    const int32_t* __restrict__ faces, const float* __restrict__ vertex_colors,
                                                    Workspace ws, Dims d)
{
    __shared__ SetupStage stages[DIRT_SETUP_THREADS / 32];
    SetupStage& st = stages[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)d.B * d.F;
    const long long gbase = gid - lane;   // the warp's first face
    if (gid == 0) ws.header->tag = workspace_tag(vertices, faces, d.B, d.H, d.W, d.V, d.F);
    if (gbase >= total) return;           // the whole warp: the lanes below stay together for the warp-wide steps
    const bool live = gid < total;
    const int b = live ? (int)(gid / d.F) : 0;
    const int f = (int)(gid - (long long)b * d.F);
    const bool shade = BIN && vertex_colors != nullptr && DIRT_SETUP_ABLATE != 2;
    AblationSink sink(ws.header);

    // what the warp-wide steps need of this lane's face
    int bin = BIN_NONE, tx0 = 0, tx1 = 0, ty0 = 0, ty1 = 0;
    bool shaded = false;

    const auto face = [&]() {
        const float* verts = vertices + (size_t)b * d.V * 4;

        // A face that cannot produce a fragment leaves a defined record (kind = culled, edge functions negative) and is not
        // binned.  Every rejection below ends here, so the path of a face that survives has no merges with default values.
        const auto cull = [&]() {
            st.cov[slot64(lane, 0)] = make_uint4(0u, 0u, 0u, 0u);                 // A0 B0 A1 B1
            st.cov[slot64(lane, 1)] = make_uint4(0u, 0u, 0u, 0u);                 // A2 B2 zA zB
            st.cov[slot64(lane, 2)] = make_uint4(~0u, ~0u, ~0u, ~0u);             // q0 = q1 = -1
            st.cov[slot64(lane, 3)] = make_uint4(~0u, ~0u, 0u, KIND_CULLED);      // q2 = -1, zC, kind
            st.itp[slot64(lane, 0)] = make_uint4(0u, 0u, 0u, 0u);
            st.itp[slot64(lane, 1)] = make_uint4(0u, 0u, 0u, 0u);
            st.itp[slot64(lane, 2)] = make_uint4(__float_as_uint(1.0f), 0u, 0u, 0u);   // sC = 1, v0..v2 = 0
            st.itp[slot64(lane, 3)] = make_uint4(0u, 0u, 0u, 0u);
            st.xy[slot32(lane, 0)] = make_uint4(0u, 0u, 0u, 0u);
            st.xy[slot32(lane, 1)] = make_uint4(0u, 0u, 0u, 0u);
        };

        int32_t vid[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) vid[k] = __ldg(&faces[(size_t)gid * 3 + k]);
        if ((unsigned)vid[0] >= (unsigned)d.V || (unsigned)vid[1] >= (unsigned)d.V || (unsigned)vid[2] >= (unsigned)d.V) { cull(); return; }

        // the vertex colours go out with the positions, so that the face waits for one round trip of gathers, not two
        // (one 16-byte row per vertex when C = 4 and the rows are 16-byte aligned)
        float col[3][4];
        if (shade) {
            const float* cols = vertex_colors + (size_t)b * d.V * d.C;
            if (d.C == 4 && ((uintptr_t)vertex_colors & 15) == 0) {
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const float4 c = __ldg(reinterpret_cast<const float4*>(cols) + vid[k]);
                    col[k][0] = c.x; col[k][1] = c.y; col[k][2] = c.z; col[k][3] = c.w;
                }
            } else {
#pragma unroll
                for (int k = 0; k < 3; ++k)
#pragma unroll
                    for (int c = 0; c < 4; ++c) col[k][c] = c < d.C ? __ldg(cols + (size_t)vid[k] * d.C + c) : 0.0f;
            }
        }

        float p[3][4];
        bool finite = true;
        int n_behind = 0;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(verts) + vid[k]);
            p[k][0] = v.x; p[k][1] = v.y; p[k][2] = v.z; p[k][3] = v.w;
            finite = finite && isfinite(v.x) && isfinite(v.y) && isfinite(v.z) && isfinite(v.w);
            if (!(v.w > 0.0f)) ++n_behind;
        }
        if (!finite || n_behind == 3) { cull(); return; }
        if (DIRT_SETUP_ABLATE == 4) {
            sink.take(make_uint4(__float_as_uint(p[0][0]) ^ __float_as_uint(p[1][1]), __float_as_uint(p[2][2]) ^ __float_as_uint(p[0][3]),
                                 __float_as_uint(p[1][3]) ^ __float_as_uint(p[2][3]), __float_as_uint(p[0][1]) ^ __float_as_uint(p[2][0])));
            if (shade)
                sink.take(make_uint4(__float_as_uint(col[0][0]) ^ __float_as_uint(col[1][1]), __float_as_uint(col[2][2]),
                                     __float_as_uint(col[0][3]) ^ __float_as_uint(col[1][3]), __float_as_uint(col[2][3])));
            return;
        }

        // S1-S3: window coordinates snapped to 1/256 px; a vertex behind the eye or outside the guard band makes the face "hard"
        bool hard = n_behind > 0;
        int32_t xi[3] = {0, 0, 0}, yi[3] = {0, 0, 0};
        if (!hard) {
            const float halfW = 0.5f * (float)d.W, halfH = 0.5f * (float)d.H;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float xn = __fdiv_rn(p[k][0], p[k][3]);
                const float yn = __fdiv_rn(p[k][1], p[k][3]);
                const float X = __fmul_rn(__fadd_rn(xn, 1.0f), halfW);
                const float Y = __fmul_rn(__fsub_rn(1.0f, yn), halfH);
                const float fx = __fmul_rn(X, 256.0f), fy = __fmul_rn(Y, 256.0f);
                if (!(fabsf(fx) <= GUARD_BAND) || !(fabsf(fy) <= GUARD_BAND)) hard = true;
                else { xi[k] = __float2int_rn(fx); yi[k] = __float2int_rn(fy); }
            }
        }

        // S6: interpolation and depth planes
        double gq[3][3], gs[3], gz[3];
        if (!exact::planes_double(p, d.ps, gq, gs, gz)) { cull(); return; }

        // S4-S5: edge functions and the pixel bounding box of a normal face; a hard face may touch any pixel
        int32_t A[3] = {0, 0, 0}, Bc[3] = {0, 0, 0};
        int64_t q_abs[3] = {-1, -1, -1};
        int cmin = 0, cmax = d.W - 1, rmin = 0, rmax = d.H - 1;
        if (!hard) {
            const int64_t ax = xi[0], ay = yi[0], bx = xi[1], by = yi[1], cx = xi[2], cy = yi[2];
            const int64_t area2 = (bx - ax) * (cy - ay) - (cx - ax) * (by - ay);
            if (area2 == 0) { cull(); return; }
            int32_t px[3] = {xi[0], xi[1], xi[2]}, py[3] = {yi[0], yi[1], yi[2]};
            if (area2 < 0) {
                int32_t t = px[1]; px[1] = px[2]; px[2] = t;
                t = py[1]; py[1] = py[2]; py[2] = t;
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int a = (k + 1) % 3, bb = (k + 2) % 3;
                const int64_t Ak = (int64_t)py[a] - py[bb];
                const int64_t Bk = (int64_t)px[bb] - px[a];
                const int64_t Ck = -(Ak * px[a] + Bk * py[a]);
                const bool tl = (Ak > 0) || (Ak == 0 && Bk > 0);
                const int64_t Cpp = 128 * (Ak + Bk) + Ck - (tl ? 0 : 1);
                A[k] = (int32_t)Ak; Bc[k] = (int32_t)Bk; q_abs[k] = Cpp >> 8;
            }
            const int32_t xmin = min(px[0], min(px[1], px[2])), xmax = max(px[0], max(px[1], px[2]));
            const int32_t ymin = min(py[0], min(py[1], py[2])), ymax = max(py[0], max(py[1], py[2]));
            cmin = max((xmin + 127) >> 8, 0); cmax = min((xmax - 128) >> 8, d.W - 1);
            rmin = max((ymin + 127) >> 8, 0); rmax = min((ymax - 128) >> 8, d.H - 1);
            if (cmin > cmax || rmin > rmax) { cull(); return; }
        }

        // The pixel under the face's vertex of largest clip w (the first of equals), clamped to the bbox: 1/clip_w is
        // smallest there, so fp32 planes re-based to it lose the least where the relative error of S would otherwise be
        // largest.  A normal face has the snapped window position already; a hard face in front of the eye (one that leaves
        // the guard band) divides, in the operation order of S3, because its G-buffer is re-based there and the oracle must
        // find the same pixel (rule S6).  A face with a vertex behind the eye keeps pixel (0,0): its S plane crosses zero
        // on screen, so no pixel is a better anchor for all of it.
        // (selected by value, not by a runtime index, which would put p / xi / yi in local memory)
        float fx = p[0][0], fy = p[0][1], fw = p[0][3];
        int fxi = xi[0], fyi = yi[0];
#pragma unroll
        for (int k = 1; k < 3; ++k)
            if (p[k][3] > fw) { fx = p[k][0]; fy = p[k][1]; fw = p[k][3]; fxi = xi[k]; fyi = yi[k]; }
        int fcol, frow;
        if (!hard) {
            fcol = min(max(fxi >> 8, cmin), cmax);
            frow = min(max(fyi >> 8, rmin), rmax);
        } else if (n_behind > 0) {
            fcol = frow = 0;
        } else {
            const float X = floorf(__fmul_rn(__fadd_rn(__fdiv_rn(fx, fw), 1.0f), 0.5f * (float)d.W));
            const float Y = floorf(__fmul_rn(__fsub_rn(1.0f, __fdiv_rn(fy, fw)), 0.5f * (float)d.H));
            fcol = !(X >= 0.0f) ? 0 : (X > (float)(d.W - 1) ? d.W - 1 : (int)X);
            frow = !(Y >= 0.0f) ? 0 : (Y > (float)(d.H - 1) ? d.H - 1 : (int)Y);
        }
        // interpolation record: planes relative to the bbox corner of a normal face; a hard face (its bbox is the frame) and
        // every shading record take the pixel above instead
        const int cref = hard ? fcol : cmin, rref = hard ? frow : rmin;
        {
            const double cr = (double)cref, rr = (double)rref;
            TriInterp itp;
            itp.q0A = (float)gq[0][0]; itp.q0B = (float)gq[0][1];
            itp.q0C = (float)__dadd_rn(__dadd_rn(__dmul_rn(gq[0][0], cr), __dmul_rn(gq[0][1], rr)), gq[0][2]);
            itp.q1A = (float)gq[1][0]; itp.q1B = (float)gq[1][1];
            itp.q1C = (float)__dadd_rn(__dadd_rn(__dmul_rn(gq[1][0], cr), __dmul_rn(gq[1][1], rr)), gq[1][2]);
            itp.sA = (float)gs[0]; itp.sB = (float)gs[1];
            itp.sC = (float)__dadd_rn(__dadd_rn(__dmul_rn(gs[0], cr), __dmul_rn(gs[1], rr)), gs[2]);
            itp.v0 = vid[0]; itp.v1 = vid[1]; itp.v2 = vid[2];
            itp.cref = cref; itp.rref = rref;
            itp.pad0 = itp.pad1 = 0;
            union { TriInterp t; uint4 u[4]; } i; i.t = itp;
#pragma unroll
            for (int c = 0; c < 4; ++c) st.itp[slot64(lane, c)] = i.u[c];
            st.xy[slot32(lane, 0)] = make_uint4(__float_as_uint(p[0][0]), __float_as_uint(p[0][1]), __float_as_uint(p[1][0]), __float_as_uint(p[1][1]));
            st.xy[slot32(lane, 1)] = make_uint4(__float_as_uint(p[2][0]), __float_as_uint(p[2][1]), 0u, 0u);
            // shading record: planes of N_c = q0*(c0 - c2) + q1*(c1 - c2) + S*c2 (q2 = S - q0 - q1), values only.  Re-based
            // to the far vertex's pixel: N_c / S is evaluated where S is small with the least rounding (w ratio 10^4 across a
            // 2048^2 face, against fp64 interpolation: 1.2-1.6x the 1e-4 bar from the bbox corner, 0.2-0.6x from there).
            if (shade) {
                const double fc = (double)fcol, fr = (double)frow;
                float4 out[4];
                out[0] = make_float4(itp.sA, itp.sB, (float)((gs[0] * fc + gs[1] * fr) + gs[2]),
                                     __uint_as_float((uint32_t)fcol | ((uint32_t)frow << 16)));
                float n[12];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const double c0 = (double)col[0][c], c1 = (double)col[1][c], c2 = (double)col[2][c];
                    const double d0 = c0 - c2, d1 = c1 - c2;
                    const double nA = gq[0][0] * d0 + gq[1][0] * d1 + gs[0] * c2;
                    const double nB = gq[0][1] * d0 + gq[1][1] * d1 + gs[1] * c2;
                    const double nC = gq[0][2] * d0 + gq[1][2] * d1 + gs[2] * c2;
                    n[3 * c] = (float)nA; n[3 * c + 1] = (float)nB; n[3 * c + 2] = (float)((nA * fc + nB * fr) + nC);
                }
                out[1] = make_float4(n[0], n[1], n[2], n[3]);
                out[2] = make_float4(n[4], n[5], n[6], n[7]);
                out[3] = make_float4(n[8], n[9], n[10], n[11]);
#pragma unroll
                for (int c = 0; c < 4; ++c) st.shade[slot64(lane, c)] = *reinterpret_cast<const uint4*>(&out[c]);
                shaded = true;
            }
        }

        // tile bounding box and the layout of the coverage record.
        // "small" faces are binned per tile and rasterised entirely in int32: that needs a bounded tile count AND bounded
        // edge coefficients (a huge, mostly off-screen face can have a small clamped bbox): |A|,|B| < 2^18, |q_rel| < 2^29
        // keep q_rel + A*dcol + B*drow (|dcol|,|drow| < 2^9 inside the binned tiles) below 2^31.
        tx0 = cmin >> TILE_W_SHIFT; tx1 = cmax >> TILE_W_SHIFT;
        ty0 = rmin >> TILE_H_SHIFT; ty1 = rmax >> TILE_H_SHIFT;
        const int64_t q0r = q_abs[0] + (int64_t)A[0] * cmin + (int64_t)Bc[0] * rmin;
        const int64_t q1r = q_abs[1] + (int64_t)A[1] * cmin + (int64_t)Bc[1] * rmin;
        const int64_t q2r = q_abs[2] + (int64_t)A[2] * cmin + (int64_t)Bc[2] * rmin;
        const int32_t cmax_abs = max(max(max(abs(A[0]), abs(Bc[0])), max(abs(A[1]), abs(Bc[1]))), max(abs(A[2]), abs(Bc[2])));
        const int64_t qlim = (int64_t)1 << 29;
        const bool small = !hard && (tx1 - tx0 + 1) * (ty1 - ty0 + 1) <= SMALL_TILE_LIMIT && cmax_abs < (1 << 18) &&
                           q0r > -qlim && q0r < qlim && q1r > -qlim && q1r < qlim && q2r > -qlim && q2r < qlim;
        {
            TriCov cov;
            cov.A0 = A[0]; cov.B0 = Bc[0]; cov.A1 = A[1]; cov.B1 = Bc[1]; cov.A2 = A[2]; cov.B2 = Bc[2];
            const float zA = (float)gz[0], zB = (float)gz[1], zC = (float)gz[2];
            if (small) {
                cov.s.kind = KIND_SMALL;
                cov.s.q0r = (int32_t)q0r; cov.s.q1r = (int32_t)q1r; cov.s.q2r = (int32_t)q2r;
                cov.s.zA = zA; cov.s.zB = zB; cov.s.zC = zC;
                cov.s.cref = cmin; cov.s.rref = rmin; cov.s.pad = 0;
            } else {
                cov.l.kind = hard ? KIND_HARD : KIND_LARGE;
                cov.l.q0 = q_abs[0]; cov.l.q1 = q_abs[1]; cov.l.q2 = q_abs[2];
                cov.l.zA = zA; cov.l.zB = zB; cov.l.zC = zC;
            }
            union { TriCov t; uint4 u[4]; } c; c.t = cov;
#pragma unroll
            for (int k = 0; k < 4; ++k) st.cov[slot64(lane, k)] = c.u[k];
        }
        bin = small ? BIN_SMALL : BIN_LARGE;
    };

    if (live) face();
    __syncwarp();
    const int nrec = (int)min(total - gbase, 32ll);   // faces of this warp

    // Binning.  A face spanning at most 2x2 tiles (nearly every face of a fine mesh) has up to four tiles, in four slots
    // (top-left, top-right, bottom-left, bottom-right); per slot the lanes naming the same tile take their positions from
    // one atomicAdd of the group's size, issued by the group's lowest lane, and all four slots' atomics go out before
    // the first result is needed.
    const bool quad = bin == BIN_SMALL && tx1 - tx0 <= 1 && ty1 - ty0 <= 1;
    const int tb = b * d.tiles;   // int32: B * tiles is (api.cu shape_ok)
    int key[4];
    unsigned peers[4];
    int base[4];
    if (BIN && DIRT_SETUP_ABLATE != 1) {
        const bool two_x = tx1 > tx0, two_y = ty1 > ty0;
        key[0] = quad ? tb + ty0 * d.tiles_x + tx0 : -1;
        key[1] = quad && two_x ? tb + ty0 * d.tiles_x + tx1 : -1;
        key[2] = quad && two_y ? tb + ty1 * d.tiles_x + tx0 : -1;
        key[3] = quad && two_x && two_y ? tb + ty1 * d.tiles_x + tx1 : -1;
#pragma unroll
        for (int k = 0; k < 4; ++k) peers[k] = __match_any_sync(0xffffffffu, key[k]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            base[k] = 0;
            if (key[k] >= 0 && lane == __ffs(peers[k]) - 1) base[k] = atomicAdd(&ws.tile_count[key[k]], __popc(peers[k]));
        }
    }

    // the records, each array in coalesced 16-byte stores (a culled face's shading record is not written)
    if (DIRT_SETUP_ABLATE != 4) {
        const auto put = [&](uint4* dst, uint4 v) {
            if (DIRT_SETUP_ABLATE == 3) sink.take(v);
            else *dst = v;
        };
        uint4* gcov = reinterpret_cast<uint4*>(ws.cov + gbase);
        uint4* gitp = reinterpret_cast<uint4*>(ws.itp + gbase);
        uint4* gxy = reinterpret_cast<uint4*>(ws.xy + gbase);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = lane + 32 * j, r = k >> 2;
            if (r < nrec) { put(gcov + k, st.cov[slot64(r, k & 3)]); put(gitp + k, st.itp[slot64(r, k & 3)]); }
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int k = lane + 32 * j, r = k >> 1;
            if (r < nrec) put(gxy + k, st.xy[slot32(r, k & 1)]);
        }
    }
    if (shade) {
        const unsigned with_shade = __ballot_sync(0xffffffffu, shaded);
        uint4* gsh = reinterpret_cast<uint4*>(ws.shade + gbase);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = lane + 32 * j, r = k >> 2;
            if ((with_shade >> r) & 1u) gsh[k] = st.shade[slot64(r, k & 3)];
        }
    }
    if (!BIN || DIRT_SETUP_ABLATE == 1) return;
    int pos[4];
    const unsigned below = (1u << lane) - 1u;
#pragma unroll
    for (int k = 0; k < 4; ++k) pos[k] = __shfl_sync(0xffffffffu, base[k], __ffs(peers[k]) - 1) + __popc(peers[k] & below);
    if (bin == BIN_NONE) return;

    const auto to_large_list = [&]() {
        const int pos = atomicAdd(&ws.large_count[b], 1);
        ws.large_list[(size_t)b * d.F + pos] = f;
    };
    const auto place = [&](int t, int pos) {
        if (pos < BIN_CAP) {
            ws.bins[((size_t)b * d.tiles + t) * BIN_CAP + pos] = f;
        } else {
            // the tile's bin is full: the overflow list of its row of tiles, and if that is full as well the large list
            // (a face that sits in both a bin and the large list is tested twice, which cannot change a minimum)
            const size_t row = (size_t)b * d.tiles_y + t / d.tiles_x;
            const int q = atomicAdd(&ws.ovf_count[row], 1);
            if (q < OVF_ROW_CAP) ws.ovf[row * OVF_ROW_CAP + q] = make_int2(t, f);
            else {
                // one byte per face, claimed with an atomic OR on the word holding it
                unsigned int* word = reinterpret_cast<unsigned int*>(ws.face_in_large) + (gid >> 2);
                const unsigned int bit = 1u << (8 * (unsigned)(gid & 3));
                if ((atomicOr(word, bit) & bit) == 0u) to_large_list();
            }
        }
    };
    if (quad) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (key[k] >= 0) place(key[k] - tb, pos[k]);
    } else if (bin == BIN_SMALL) {
        for (int ty = ty0; ty <= ty1; ++ty)
            for (int tx = tx0; tx <= tx1; ++tx) {
                const int t = ty * d.tiles_x + tx;
                place(t, atomicAdd(&ws.tile_count[tb + t], 1));
            }
    } else {
        to_large_list();
    }
}

static unsigned setup_blocks(long long total)
{
    return (unsigned)max((total + DIRT_SETUP_THREADS - 1) / DIRT_SETUP_THREADS, 1ll);
}

cudaError_t launch_setup_and_bin(const float* vertices, const int32_t* faces, const float* vertex_colors, const Workspace& ws,
                                 const Dims& d, cudaStream_t stream)
{
    if (!shade_records_ok(d)) vertex_colors = nullptr;
    const long long total = (long long)d.B * d.F;
    cudaError_t e;
    if ((e = cudaMemsetAsync(ws.tile_count, 0, ws.zero_bytes, stream)) != cudaSuccess) return e;
    // at least one block, even without faces: its first thread leaves the tag, which a later call reusing the workspace checks
    ScopedKernelTimer timer(3, stream);
    setup_kernel<true><<<setup_blocks(total), DIRT_SETUP_THREADS, 0, stream>>>(vertices, faces, vertex_colors, ws, d);
    return launched();
}

cudaError_t launch_setup_only(const float* vertices, const int32_t* faces, const Workspace& ws, const Dims& d,
                              cudaStream_t stream)
{
    const long long total = (long long)d.B * d.F;
    cudaError_t e;
    if ((e = cudaMemsetAsync(ws.header, 0, sizeof(Header), stream)) != cudaSuccess) return e;
    ScopedKernelTimer timer(3, stream);
    setup_kernel<false><<<setup_blocks(total), DIRT_SETUP_THREADS, 0, stream>>>(vertices, faces, nullptr, ws, d);
    return launched();
}

}  // namespace dirt
