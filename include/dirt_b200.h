/*
 * dirt_b200.h -- C ABI of libdirt_b200.so, the sm_90a replacement for the
 * `Rasterise` / `RasteriseGrad` custom ops of pmh47/dirt.
 *
 * Every entry point takes plain device pointers and sizes (no torch / TF types),
 * enqueues all its work on the CUDA stream it is given, never synchronises the
 * host, never allocates device memory and keeps no global state.  The caller
 * owns every buffer, including the workspace.
 *
 * Reference interfaces replaced (paths relative to the reference checkout):
 *   dirt_rasterise_forward   <- REGISTER_OP("Rasterise") + RasteriseOpGpu::Compute
 *                               csrc/rasterise_egl.cpp:32-51, 276-408
 *   dirt_rasterise_backward  <- REGISTER_OP("RasteriseGrad") + RasteriseGradOpGpu::Compute
 *                               csrc/rasterise_grad_egl.cpp:33-53, 324-485 and the kernel
 *                               assemble_grads, csrc/rasterise_grad_egl.cu:93-236
 *   dirt_rasterise_visibility<- the backward G-buffer (barycentrics, clip-w, indices) that
 *                               the reference renders with GL, csrc/shaders.cpp:45-79,
 *                               csrc/rasterise_grad_egl.cpp:432-456 (debug / parity tests)
 *   height/width/channels    <- the HWC op attributes, csrc/hwc.h:7-30
 *
 * Layouts (all row-major, channels last, row 0 = top of the image = clip-space y=+1,
 * csrc/rasterise_egl.cu:23,80):
 *   background, pixels, grad_pixels, grad_background : float32 [B, H, W, C]
 *   vertices, grad_vertices                          : float32 [B, V, 4]   (clip space x,y,z,w)
 *   vertex_colors, grad_vertex_colors                : float32 [B, V, C]
 *   faces                                            : int32   [B, F, 3]
 *   face_ids                                         : int32   [B, H, W]   (-1 = background)
 *   gbuffer                                          : float32 [B, H, W, 4] (bary0, bary1, bary2, clip_w;
 *                                                      (-1,-1,-1,+inf) where uncovered)
 */
#ifndef DIRT_B200_H
#define DIRT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Error codes: 0 on success, negative on failure.  Nothing aborts the process
 * (the reference LOG(FATAL)s on every CUDA/GL error, csrc/rasterise_egl.cpp:82-86). */
enum {
    DIRT_OK = 0,
    DIRT_ERR_BAD_SHAPE = -1,        /* B,H,W,C,V,F out of range (csrc/hwc.h:27-28; rasterise_egl.cpp:301-316) */
    DIRT_ERR_NULL_POINTER = -2,
    DIRT_ERR_WORKSPACE_TOO_SMALL = -3,
    DIRT_ERR_BAD_CHANNEL_GROUPS = -4, /* groups must be 1 or 3 wide and sum to C (rasterise_ops.py:80-108) */
    DIRT_ERR_TOO_MANY_VERTICES = -5,  /* V > 2^24, csrc/rasterise_grad_egl.cpp:399-405 */
    DIRT_ERR_CUDA = -6,               /* a CUDA runtime call or kernel launch failed */
    DIRT_ERR_MISALIGNED = -7,         /* a pointer is not aligned as required (workspace: 256 B, tensors: 4 B) */
    DIRT_ERR_STALE_WORKSPACE = -8     /* dirt_workspace_status: a backward call was promised setup records that were not there */
};

/* Human-readable text for an error code (static storage, never NULL). */
const char* dirt_error_string(int code);

/* Library / ABI version, bumped whenever a signature changes. */
int dirt_abi_version(void);

/* Bytes of device workspace that forward / backward / visibility need for these sizes.
 * Deterministic function of the sizes only (no data dependence, no host sync):
 * triangle records + bounded per-tile reference lists + per-tile counters. */
size_t dirt_workspace_bytes(int B, int H, int W, int C, int V, int F);

/* The same without the B*H*W*4-byte block that only a backward call WITHOUT face ids uses (it derives them there):
 * enough for forward, visibility, and every backward call that is handed the forward's face ids. */
size_t dirt_workspace_bytes_min(int B, int H, int W, int C, int V, int F);

/* Forward: pixels = rasterise(background, vertices, vertex_colors, faces).
 * Handles any C >= 1 in one pass (the reference runs one op per channel group of 3 or 1,
 * rasterise_ops.py:86-108; the forward result does not depend on the grouping).
 * face_ids_out may be NULL; when given it receives the per-pixel visible face index,
 * which dirt_rasterise_backward accepts back to skip re-deriving visibility. */
int dirt_rasterise_forward(const float* background, const float* vertices,
                           const float* vertex_colors, const int32_t* faces,
                           float* pixels, int32_t* face_ids_out,
                           int B, int H, int W, int C, int V, int F,
                           void* workspace, size_t workspace_bytes, void* cuda_stream);

/* Backward: the RasteriseGrad op.  `pixels` is an input (deferred shading passes shaded
 * pixels, rasterise_ops.py:206-210).  channel_groups (host pointer) lists the widths of the
 * reference's channel groups, e.g. {3,1} for C=4; each group takes its own Scharr / dilation
 * decision and grad_vertices is summed over groups (rasterise_ops.py:163).  NULL/0 means the
 * reference's own greedy split of C.
 * face_ids may be NULL: visibility is then re-derived from (vertices, faces) inside the call.
 * workspace_holds_setup != 0 promises that `workspace` is the buffer a preceding dirt_rasterise_forward /
 * dirt_rasterise_visibility call on the SAME (vertices, faces, H, W) filled and that nothing has written to it
 * since: the per-face setup records are then reused instead of recomputed (only meaningful with face_ids).
 * The promise is checked on the device: the setup pass leaves a tag (hash of the vertices / faces pointers and the
 * sizes) in the workspace; a backward call that finds another tag sets an error flag in the workspace (reported by
 * dirt_workspace_status) and writes NaN into grad_vertices[0] instead of returning plausible numbers.  What the tag
 * cannot see is an in-place change of the vertex VALUES between the two calls; the Python layer covers that with
 * the tensors' version counters.
 * grad_vertices / grad_vertex_colors are zeroed by the library before accumulation;
 * grad_background is written exactly once per pixel. */
int dirt_rasterise_backward(const float* vertices, const int32_t* faces,
                            const float* pixels, const float* grad_pixels,
                            const int32_t* face_ids,
                            float* grad_background, float* grad_vertices, float* grad_vertex_colors,
                            int B, int H, int W, int C, int V, int F,
                            const int* channel_groups, int n_groups, int workspace_holds_setup,
                            void* workspace, size_t workspace_bytes, void* cuda_stream);

/* dirt_rasterise_backward with options (flags = 0 is dirt_rasterise_backward itself):
 *  DIRT_BWD_SHARED_GEOMETRY  the vertex gradients are ACCUMULATED OVER THE BATCH: grad_vertices is [V,4] and
 *      grad_vertex_colors [V,C], sum_b of the per-item results -- the gradient of geometry / colours that are parameters
 *      shared by the batch (SURVEY 8e; the reference leaves that sum to TensorFlow's broadcast gradient).  Saves the
 *      [B,V,.] buffers, their memsets and the reduction pass; it is the buffer a multi-GPU job all-reduces.
 *  DIRT_BWD_SKIP_POSITION    grad_vertices is not computed (left zero): no Scharr filter, no dilation, `pixels` is not read.
 *  DIRT_BWD_SKIP_COLOUR      grad_vertex_colors is not computed (left zero) and grad_background is not written.
 *  The two SKIP flags serve deferred shading, whose gradient is two RasteriseGrad calls of which only one output each
 *  is used (dirt/rasterise_ops.py:206-237: vertices from the shaded pixels, attributes / background from the G-buffer). */
enum {
    DIRT_BWD_SHARED_GEOMETRY = 1,
    DIRT_BWD_SKIP_POSITION = 2,
    DIRT_BWD_SKIP_COLOUR = 4
};
int dirt_rasterise_backward_ex(const float* vertices, const int32_t* faces,
                               const float* pixels, const float* grad_pixels,
                               const int32_t* face_ids,
                               float* grad_background, float* grad_vertices, float* grad_vertex_colors,
                               int B, int H, int W, int C, int V, int F,
                               const int* channel_groups, int n_groups, int workspace_holds_setup, int flags,
                               void* workspace, size_t workspace_bytes, void* cuda_stream);

/* dirt_rasterise_backward_ex with reproducible results (DESIGN.md §7.4): the same arguments, flags, channel groups and
 * outputs, the same per-pixel terms and dilation decisions, but no float atomics.  Each vertex gradient is one float64
 * sum in a fixed order (pixels of a face in raster order, then the face corners of the vertex in ascending id k*F + f,
 * then the items in order under DIRT_BWD_SHARED_GEOMETRY), rounded once to fp32.  Two calls on the same inputs give
 * bit-identical outputs.  An item's gradients do not depend on the other items of the batch, except where a 1-wide
 * channel group's Scharr taps at the end of an image read the next image's first pixels in flat order (the reference's
 * semantics, as in dirt_rasterise_backward_ex); with groups of width 3 only they never do.  Needs 3*B*F < 2^31.
 *
 * scratch: at least dirt_rasterise_backward_deterministic_bytes(B, H, W, C, V, F) bytes, 256-byte aligned, owned by the
 * caller and separate from the workspace (which means what it means for dirt_rasterise_backward_ex).  Nothing in it needs
 * to be initialised.  After the call it starts with the dilation codes: C planes of B*H*W bytes, plane g (g < the number
 * of channel groups) holding group g's code per pixel, in [B][H][W] order:
 *   bits 0-1  0: no position term, 1: the pixel's own face takes it, 2: the neighbour one step along the preferred
 *             direction does (the dilation took it), 3: the neighbour one step against it does;
 *   bit 2     the preferred step runs along the row (the Scharr x sum dominates); meaningful for codes 2 and 3.
 * The step is +1 along the axis (column + 1, or the row above) on pixels whose col + row is even, -1 on odd ones.
 * Returns 0 for B == 0; the size is a function of the shapes alone (SIZE_MAX if it does not fit a size_t). */
size_t dirt_rasterise_backward_deterministic_bytes(int B, int H, int W, int C, int V, int F);
int dirt_rasterise_backward_deterministic(const float* vertices, const int32_t* faces,
                                          const float* pixels, const float* grad_pixels,
                                          const int32_t* face_ids,
                                          float* grad_background, float* grad_vertices, float* grad_vertex_colors,
                                          int B, int H, int W, int C, int V, int F,
                                          const int* channel_groups, int n_groups, int workspace_holds_setup, int flags,
                                          void* workspace, size_t workspace_bytes, void* scratch, size_t scratch_bytes,
                                          void* cuda_stream);

/* Waits for the stream and reports whether a backward call found the workspace not to hold the setup records it was
 * promised (DIRT_ERR_STALE_WORKSPACE), else DIRT_OK.  The only entry point that synchronises the host. */
int dirt_workspace_status(const void* workspace, size_t workspace_bytes,
                          int B, int H, int W, int C, int V, int F, void* cuda_stream);

/* Debug / parity: the visibility G-buffer alone (either output may be NULL). */
int dirt_rasterise_visibility(const float* vertices, const int32_t* faces,
                              int32_t* face_ids, float* gbuffer,
                              int B, int H, int W, int V, int F,
                              void* workspace, size_t workspace_bytes, void* cuda_stream);

/* Screen-space derivatives of G-buffer attributes (DESIGN.md §7.7), e.g. uv footprints for a trilinear texture lookup.
 *   attributes   float32 [B, V, C]: the vertex attributes of a forward call (its vertex_colors)
 *   face_ids     int32 [B, H, W]: that call's face_ids_out (required)
 *   derivatives  float32 [B, H, W, 2, channel_count]: for channels c in [first_channel, first_channel + channel_count),
 *                index 0 of the `2` axis is d a_c / dx (x along W, to the right), index 1 d a_c / dy (y along H,
 *                downwards), in attribute units per pixel at the pixel centre, a_c being the perspective-correct
 *                interpolant of the attributes of the face the pixel shows.  A pixel whose id is not in [0, F) gets 0.
 * The values come from the face's interpolation planes in the workspace (the G-buffer's own), with b_k = q_k / S:
 *   d a / dx = ((a0 - a2) (q0A - b0 sA) + (a1 - a2) (q1A - b1 sA)) / S, and the same with the B coefficients for y.
 * No gradient, no atomics: two calls on the same inputs give bit-identical outputs.
 * workspace_holds_setup means what it means for dirt_rasterise_backward: != 0 reuses the setup records of the forward
 * call on the same (vertices, faces, H, W) in `workspace` (checked on the device; a workspace of other geometry sets the
 * error dirt_workspace_status reports and every output is NaN); 0 recomputes them there first.
 * An empty channel range or one outside [0, C) is DIRT_ERR_BAD_SHAPE.  B = 0: nothing is launched.  All pointers 4-byte
 * aligned (vertices 16); derivatives 8- (one channel) or 16-byte aligned (two or four) enable the vector stores.  Only
 * enqueues work on cuda_stream. */
int dirt_rasterise_derivatives(const float* vertices, const int32_t* faces, const float* attributes,
                               const int32_t* face_ids, float* derivatives,
                               int B, int H, int W, int C, int V, int F,
                               int first_channel, int channel_count,
                               int workspace_holds_setup, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* Multi-GPU (one process per GPU, one node): sum over the ranks of the batch-shared vertex gradient -- the [V,4 | V,C] buffer
 * a DIRT_BWD_SHARED_GEOMETRY call fills -- over peer memory, as ONE kernel of `world` CTAs per rank and step: every rank
 * pushes its buffer into its slot of every peer's exchange area (stores through the NVLink peer mapping), releases a flag
 * there, waits for the `world` flags of its own area and adds its slots in rank order into `out` (bit-identical on all
 * ranks).  The reference has no counterpart (no multi-GPU path: tests/multi_gpu_test.py); TensorFlow users would all-reduce
 * the op's gradient outside it.
 *   dirt_peer_exchange_bytes  size of one rank's exchange area for buffers of `count` floats (two step parities x world slots).
 *   peer_slots[p] / peer_flags[p]  HOST arrays of `world` DEVICE pointers: rank p's exchange area / its flag words
 *                                  (2*world uint32, zero before the first call) as mapped into THIS process (own rank
 *                                  included).  The mapping itself (cudaIpc / VMM handles) is the caller's plumbing.
 *   sequence  1, 2, 3, ... : the same value on every rank for the same step; consecutive calls on one stream.
 *   local != out, both 16-byte aligned, count a multiple of 4.  Only enqueues work on cuda_stream. */
size_t dirt_peer_exchange_bytes(int world, long long count);
int dirt_peer_exchange(const float* local, float* out, void* const* peer_slots, void* const* peer_flags,
                       int world, int rank, long long count, unsigned int sequence, void* cuda_stream);

/* Differentiable texture lookup: the bilinear / nearest lookup of the reference's textured sample
 * (samples/textured.py:30-60), with the four bilinear texels wrapping around the texture edge.
 *   texture          float32 [TB, TH, TW, C]: TB = 1 (one texture shared by every lookup) or TB = B (one per batch item)
 *   indices          float32 [B, N, 2]: fractional (row, column) texel indices; (0, 0) is the top-left texel corner
 *   out, grad_out    float32 [B, N, C]
 *   grad_texture     float32 [TB, TH, TW, C]; grad_indices float32 [B, N, 2]
 *   mode DIRT_TEXTURE_BILINEAR: r0 = floor(row) mod TH, c0 = floor(col) mod TW, r1 = (r0+1) mod TH, c1 = (c0+1) mod TW
 *        (mod with the sign of the divisor), fr / fc = index - floor(index), and
 *        out = t00*(1-fc)*(1-fr) + t01*fc*(1-fr) + t10*(1-fc)*fr + t11*fc*fr, each operation rounded as written, left to
 *        right, in fp32: bit-identical to the same expression evaluated by torch.
 *   mode DIRT_TEXTURE_NEAREST: the texel at (trunc(row), trunc(col)), each clamped to the texture; no index gradient.
 * A lookup with a non-finite index returns 0 in every channel, reads no texel and contributes no gradient.
 * Backward: grad_texture is zeroed by the library before it accumulates into it; grad_indices is written once per
 * lookup (through the fractions only; zero for nearest).  Either may be NULL, and that half of the work is skipped;
 * texture may then be NULL unless grad_indices of a bilinear lookup is wanted.
 * B = 0 or N = 0: nothing is launched (the backward call still zeroes grad_texture).  All pointers 4-byte aligned;
 * 8- / 16-byte alignment enables the vector paths. */
enum {
    DIRT_TEXTURE_BILINEAR = 0,
    DIRT_TEXTURE_NEAREST = 1
};
int dirt_texture_sample(const float* texture, const float* indices, float* out,
                        int TB, int TH, int TW, int C, int B, long long N, int mode, void* cuda_stream);
int dirt_texture_sample_backward(const float* texture, const float* indices, const float* grad_out,
                                 float* grad_texture, float* grad_indices,
                                 int TB, int TH, int TW, int C, int B, long long N, int mode, void* cuda_stream);

/* dirt_texture_sample_backward with a reproducible grad_texture (DESIGN.md §7.5): the same arguments, NULL and alignment
 * rules and outputs; grad_indices is the same, bit for bit.  grad_texture has no float atomics: each (texel, channel) is
 * one float64 sum, rounded once to fp32, of the terms grad_out[g][ch] * w (the fp32 product, w the corner's bilinear
 * weight, 1 for nearest; a zero weight adds +0.0; a lookup with a non-finite index adds nothing).  Texel (r, c) of
 * texture tb takes, in this order, the corner-00 terms of the lookups whose base texel (r0, c0) is (r, c), the corner-01
 * terms of those based at (r, c-1), corner 10 from (r-1, c) and corner 11 from (r-1, c-1), modulo the texture size
 * (nearest: the one texel read); within a corner, the lookups go in ascending id g = b*N + n.  The L terms of that
 * sequence are cut into chunks of 4096: in each, lane t of 32 sums the terms t, t + 32, ... of the chunk in order from
 * +0.0, the 32 sums meet in the xor butterfly over lane offsets 16, 8, 4, 2, 1, and the chunk sums are added in chunk
 * order from +0.0.  Two calls on the same inputs give bit-identical outputs; with per-item textures (TB = B) an item's
 * grad_texture does not depend on the other items.  Needs B*N < 2^31 and TB*TH*TW < 2^31 - 1 (else DIRT_ERR_BAD_SHAPE).
 * scratch: at least dirt_texture_sample_backward_deterministic_bytes(...) bytes, 256-byte aligned, owned by the caller,
 * needing no initialisation; it may be NULL when grad_texture is NULL or there are no lookups.  The size is a function of
 * the shapes alone (0 for no lookups or shapes this entry rejects): 16 bytes per lookup for the sort, 4 per texel for the
 * segment offsets, the sort's digit counts and the chunk sums of long sequences. */
size_t dirt_texture_sample_backward_deterministic_bytes(int TB, int TH, int TW, int C, int B, long long N, int mode);
int dirt_texture_sample_backward_deterministic(const float* texture, const float* indices, const float* grad_out,
                                               float* grad_texture, float* grad_indices,
                                               int TB, int TH, int TW, int C, int B, long long N, int mode,
                                               void* scratch, size_t scratch_bytes, void* cuda_stream);

/* Mipmapped (trilinear) texture lookup (DESIGN.md §7.6), with gradients to the texels and to the indices.
 * Levels: level 0 is the texture [TB, TH, TW, C]; level k+1 exists while level k has both dimensions even, and is its
 * 2x2 box mean per channel, ((t[2i][2j] + t[2i][2j+1]) + (t[2i+1][2j] + t[2i+1][2j+1])) * 0.25, each operation rounded
 * in that order in fp32.  Level k is [TB, TH >> k, TW >> k, C].  The pyramid buffer packs levels 1 .. L-1 in that order
 * (level 0 is not copied); a texture with an odd dimension has L = 1 and an empty pyramid.
 * Index mapping: texel j of a level has its full bilinear weight at index j, so level k >= 1 is read at
 * (index + 0.5) * 2^-k - 0.5, each operation rounded in fp32 in that order, and level 0 at the index itself; each read
 * is the bilinear lookup of DIRT_TEXTURE_BILINEAR at that level's size (wrapping around its edges).
 * Level of detail: derivatives float32 [B, N, 4] = (d row / dx, d col / dx, d row / dy, d col / dy) in level-0 texels
 * per pixel; rho^2 = max(d0^2 + d1^2, d2^2 + d3^2) (NaN if either sum is NaN), lambda = 0.5 * log2(rho^2), NaN -> 0,
 * clamped to [0, L-1]; l = floor(lambda), f = lambda - l, and out = (1-f) * bilinear_l + f * bilinear_{l+1}, each
 * operation rounded in that order.  f == 0 reads level l alone and returns it exactly: every lookup with rho <= 1 equals
 * the bilinear lookup bit for bit.
 * Gradients: to the texture through both levels' bilinear weights, then the pyramid's adjoint (a level-k texel passes
 * 0.25 x its gradient to each of its four children); to the indices through both levels' fractions, scaled by 2^-k.
 * The derivatives get none.  A lookup with a non-finite index returns 0, reads nothing and passes no gradient.
 *   dirt_texture_mip_levels         L for a TH x TW texture (0 if either is not positive).
 *   dirt_texture_mip_pyramid_bytes  size of the pyramid buffer (0 when L = 1 or for a bad shape).
 *   dirt_texture_mip_build          writes the pyramid from the texture: one launch per level 1 .. L-1.
 *   dirt_texture_sample_trilinear   the forward lookup; pyramid may be NULL when L = 1.
 *   dirt_texture_sample_trilinear_backward  grad_texture is zeroed by the library before it accumulates; grad_indices
 *       is written once per lookup.  Either may be NULL, and that half of the work is skipped; texture and pyramid are
 *       read only for grad_indices.  deterministic != 0: grad_texture is bit-reproducible (each level's gradient by the
 *       path of dirt_texture_sample_backward_deterministic, then the fixed-order adjoint; DESIGN.md §7.6), with that
 *       path's limits (B*N < 2^31, TB*TH*TW < 2^31 - 1, else DIRT_ERR_BAD_SHAPE).  scratch: at least
 *       dirt_texture_sample_trilinear_backward_bytes(...) bytes, 256-byte aligned, owned by the caller, needing no
 *       initialisation; a function of the shapes alone, 0 (and scratch may be NULL) when grad_texture needs none.
 *       scratch is read only when grad_texture is wanted and there are lookups.
 * B = 0 or N = 0: nothing is launched (the backward call still zeroes grad_texture).  All pointers 4-byte aligned;
 * 8-byte indices, 16-byte derivatives and row-aligned texture, pyramid, outputs enable the vector paths. */
int dirt_texture_mip_levels(int TH, int TW);
size_t dirt_texture_mip_pyramid_bytes(int TB, int TH, int TW, int C);
int dirt_texture_mip_build(const float* texture, float* pyramid, int TB, int TH, int TW, int C, void* cuda_stream);
int dirt_texture_sample_trilinear(const float* texture, const float* pyramid, const float* indices,
                                  const float* derivatives, float* out,
                                  int TB, int TH, int TW, int C, int B, long long N, void* cuda_stream);
size_t dirt_texture_sample_trilinear_backward_bytes(int TB, int TH, int TW, int C, int B, long long N, int deterministic);
int dirt_texture_sample_trilinear_backward(const float* texture, const float* pyramid, const float* indices,
                                           const float* derivatives, const float* grad_out,
                                           float* grad_texture, float* grad_indices,
                                           int TB, int TH, int TW, int C, int B, long long N, int deterministic,
                                           void* scratch, size_t scratch_bytes, void* cuda_stream);

/* Seamless cube-map lookup (DESIGN.md §7.10), with gradients to the texels and to the directions.
 *   cubemap          float32 [TB, 6, S, S, C], faces +X, -X, +Y, -Y, +Z, -Z; TB = 1 (shared) or TB = B (one per item)
 *   directions       float32 [B, N, 3], any length; out, grad_out float32 [B, N, C]
 *   grad_cubemap     float32 [TB, 6, S, S, C]; grad_directions float32 [B, N, 3]
 *   atlas            the padded faces [6, TB, S+2, S+2, C], dirt_cubemap_atlas_bytes(TB, S, C) bytes, written by
 *                    dirt_cubemap_sample and read by dirt_cubemap_sample_backward (grad_directions of a bilinear lookup)
 * Face: the component of largest magnitude (ties to x over y over z), with the OpenGL table of (sc, tc, ma):
 * +X (-z, -y), -X (z, -y), +Y (x, z), -Y (x, -z), +Z (x, -y), -Z (-x, -y), ma = |major component|;
 * s = (sc / ma + 1) * 0.5, t = (tc / ma + 1) * 0.5, each operation rounded in fp32 in that order.
 *   mode DIRT_TEXTURE_BILINEAR: the bilinear rule of dirt_texture_sample on face f's padded face at
 *        ((t * S - 0.5) + 1, (s * S - 0.5) + 1).  A border texel beside an edge is the adjacent face's texel that
 *        holds the projection of the direction through its centre; a border corner is ((own corner texel + row
 *        neighbour) + column neighbour) / 3.  So a lookup within half a texel of an edge blends the adjacent face.
 *   mode DIRT_TEXTURE_NEAREST: face texel (clamp(floor(t * S), 0, S-1), clamp(floor(s * S), 0, S-1)); no direction
 *        gradient.
 * A zero or non-finite direction returns 0 in every channel, reads no texel and contributes no gradient.
 * Backward: grad_cubemap is written in full (zeroed for no lookups); grad_directions is written once per lookup.
 * Either may be NULL, and that half of the work is skipped.  deterministic != 0: grad_cubemap is bit-reproducible
 * (per face, the path of dirt_texture_sample_backward_deterministic over that face's padded block, then the border's
 * fixed-order adjoint), with that path's limits (B*N < 2^31, TB*(S+2)^2 < 2^31 - 1, else DIRT_ERR_BAD_SHAPE); an item's
 * gradient then does not depend on the other items.  scratch: at least dirt_cubemap_sample_backward_bytes(...) bytes,
 * 256-byte aligned, owned by the caller, needing no initialisation, a function of the shapes alone; read only when
 * grad_cubemap is wanted and there are lookups (it may be NULL otherwise).
 * S in 1 .. 2^14.  B = 0 or N = 0: nothing is launched (the backward call still zeroes grad_cubemap).  All pointers
 * 4-byte aligned; row-aligned atlas, out, grad_out enable the vector paths. */
size_t dirt_cubemap_atlas_bytes(int TB, int S, int C);
int dirt_cubemap_sample(const float* cubemap, const float* directions, float* atlas, float* out,
                        int TB, int S, int C, int B, long long N, int mode, void* cuda_stream);
size_t dirt_cubemap_sample_backward_bytes(int TB, int S, int C, int B, long long N, int mode, int deterministic);
int dirt_cubemap_sample_backward(const float* atlas, const float* directions, const float* grad_out,
                                 float* grad_cubemap, float* grad_directions,
                                 int TB, int S, int C, int B, long long N, int mode, int deterministic,
                                 void* scratch, size_t scratch_bytes, void* cuda_stream);

/* Mipmapped (trilinear) cube-map lookup (DESIGN.md §7.11), with gradients to the texels, the directions and the level
 * of detail.  Shapes, faces and the per-level lookup as for dirt_cubemap_sample's bilinear mode, and:
 *   lod              float32 [B, N], the level of detail in levels, 0 the finest; grad_lod float32 [B, N]
 *   atlas            the padded faces of every level, dirt_cubemap_mip_atlas_bytes(TB, S, C) bytes, written by
 *                    dirt_cubemap_sample_trilinear; the only state dirt_cubemap_sample_trilinear_backward reads
 * Levels: L = dirt_texture_mip_levels(S, S); level k >= 1 is each face's 2x2 box mean of level k-1 (S >> k per edge),
 * bit for bit dirt_texture_mip_build of the [6*TB, S, S, C] faces.  Level k is read at ((t * S_k - 0.5) + 1,
 * (s * S_k - 0.5) + 1) on its own padded faces (S_k = S >> k), whose border comes from the adjacent faces at level k.
 * lambda = lod, NaN -> 0, clamped to [0, L-1]; l = floor(lambda), f = lambda - l;
 * out = (1-f) * b_l + f * b_{l+1}, each operation rounded in that order, and b_l alone (level l+1 not read) when
 * f == 0: lod <= 0 is dirt_cubemap_sample's bilinear lookup bit for bit.
 * Backward: grad_cubemap through both levels' weights, each level's border adjoint and the pyramid's adjoint;
 * grad_directions through both levels' fractions; grad_lod = sum_c grad_out_c * (b_{m+1,c} - b_{m,c}),
 * m = min(floor(lambda), L-2), and 0 where lod < 0, lod > L-1, lod is NaN, L = 1 or the direction is invalid.
 * Any of the three may be NULL, and its work is skipped.  deterministic != 0: grad_cubemap is bit-reproducible (per
 * level and face, the path of dirt_texture_sample_backward_deterministic, then the fixed-order adjoints), with the
 * limits of dirt_cubemap_sample_backward's deterministic path.  scratch as for dirt_cubemap_sample_backward, at least
 * dirt_cubemap_sample_trilinear_backward_bytes(...) bytes.  B = 0 or N = 0: nothing is launched (the backward call
 * still zeroes grad_cubemap). */
size_t dirt_cubemap_mip_atlas_bytes(int TB, int S, int C);
int dirt_cubemap_sample_trilinear(const float* cubemap, const float* directions, const float* lod, float* atlas,
                                  float* out, int TB, int S, int C, int B, long long N, void* cuda_stream);
size_t dirt_cubemap_sample_trilinear_backward_bytes(int TB, int S, int C, int B, long long N, int deterministic);
int dirt_cubemap_sample_trilinear_backward(const float* atlas, const float* directions, const float* lod,
                                           const float* grad_out, float* grad_cubemap, float* grad_directions,
                                           float* grad_lod, int TB, int S, int C, int B, long long N, int deterministic,
                                           void* scratch, size_t scratch_bytes, void* cuda_stream);

/* Split-sum GGX image-based lighting (DESIGN.md §7.12).  Shapes as for dirt_cubemap_sample_trilinear, and:
 *   atlas            dirt_cubemap_ggx_atlas_bytes(TB, S, C) bytes, 16-byte aligned: the mip atlas of the prefiltered
 *                    levels, then (float offsets) the prefiltered levels 1 .. L-1 in the layout of
 *                    dirt_texture_mip_build's pyramid of the [6*TB, S, S, C] faces, their normalisers W in the pyramid
 *                    layout of 6 faces of 1 channel (shared by every item), the texel table (one float4 per texel
 *                    of levels 0 .. L-1 of the 6 faces: direction, solid angle) and the cone table (one float4 per
 *                    16 x 16 block of those faces: axis, half-angle).  The offsets are pure functions of
 *                    (TB, S, C): DESIGN.md §7.12.
 * Levels: L = dirt_texture_mip_levels(S, S); level 0 is the cube map; level k >= 1 (S >> k per edge, roughness
 * r = k / (L-1), alpha2 = max(r, 0.045)^4) is P_k(r) = sum_j w_j src_j / W(r), w_j = D(c_j) c_j Omega_j,
 * D(c) = alpha2 / (pi k^2), k = alpha2 + (1-c)(1-alpha2)/2, c_j the fp32 cosine between the texel directions, over the
 * texels j of box level min(k, s*) (s* the coarsest level of at least 16 texels per edge, 0 when S < 16) with c_j > 0
 * and c_j >= c_k = max(0, 1 - 2 (sqrt(1000) - 1) alpha2 / (1 - alpha2)).
 * dirt_cubemap_ggx_prefilter writes the texel table, levels 1 .. L-1 and W (and uses level 0's slot of the mip atlas
 * as scratch); dirt_cubemap_sample_ggx calls it, builds the mip atlas of the levels and looks up as
 * dirt_cubemap_sample_trilinear does on them.  The backward pass reads the atlas alone: the lookup's gradients as
 * dirt_cubemap_sample_trilinear_backward's, then the prefilter's adjoint (a gather over the same pairs, no atomics)
 * and the box pyramid's.  scratch: dirt_cubemap_sample_ggx_backward_bytes bytes, 256-byte aligned, when grad_cubemap
 * is given and B*N > 0. */
size_t dirt_cubemap_ggx_atlas_bytes(int TB, int S, int C);
int dirt_cubemap_ggx_prefilter(const float* cubemap, float* atlas, int TB, int S, int C, void* cuda_stream);
int dirt_cubemap_sample_ggx(const float* cubemap, const float* directions, const float* lod, float* atlas, float* out,
                            int TB, int S, int C, int B, long long N, void* cuda_stream);
size_t dirt_cubemap_sample_ggx_backward_bytes(int TB, int S, int C, int B, long long N, int deterministic);
int dirt_cubemap_sample_ggx_backward(const float* atlas, const float* directions, const float* lod, const float* grad_out,
                                     float* grad_cubemap, float* grad_directions, float* grad_lod, int TB, int S, int C,
                                     int B, long long N, int deterministic, void* scratch, size_t scratch_bytes,
                                     void* cuda_stream);
/* The split-sum BRDF table, float32 [N, N, 2] = (A, B) at n.v = (i + 0.5) / N (row i) and roughness (j + 0.5) / N
 * (column j): A = integral of (1 - F_c) D Vis (n.l), B = of F_c D Vis (n.l) over light directions, F_c = (1 - v.h)^5,
 * D and Vis those of dirt_ggx_lighting_forward; a fixed midpoint rule in float64 over the GGX half-vector
 * distribution.  N <= 4096. */
int dirt_ggx_brdf_table(float* table, int N, void* cuda_stream);
/* Order-2 SH projection of cube maps, cubemap float32 [TB, 6, S, S, C] -> coeffs float32 [TB, 9, C]:
 * L_k = sum_j L(l_j) Y_k(l_j) Omega_j over the texels j with the texel table's direction and solid angle (level 0 of
 * dirt_cubemap_ggx_prefilter's table), Y the real order-2 basis of dirt_sh_lighting_forward.  Per item and chunk of
 * texels the sums are float64 in a fixed order, then added over the chunks in order and rounded once: bit-reproducible.
 * The backward pass writes grad_cubemap = Omega_j sum_k Y_k(l_j) grad_coeffs_k in full.  scratch:
 * dirt_cubemap_sh_project_bytes(TB, S, C) bytes, 256-byte aligned (the texel table and the partial sums). */
size_t dirt_cubemap_sh_project_bytes(int TB, int S, int C);
int dirt_cubemap_sh_project(const float* cubemap, float* coeffs, void* scratch, size_t scratch_bytes, int TB, int S, int C,
                            void* cuda_stream);
int dirt_cubemap_sh_project_backward(const float* grad_coeffs, float* grad_cubemap, void* scratch, size_t scratch_bytes,
                                     int TB, int S, int C, void* cuda_stream);

/* Equirectangular (latitude-longitude) panoramas to cube maps (DESIGN.md §7.13), panorama float32 [TB, H, W, C] ->
 * cubemap float32 [TB, 6, S, S, C] (faces and orientation as for dirt_cubemap_sample), with the adjoint.
 * Panorama row 0 is the zenith (+Y); texel (r, c) is centred at theta = (r + 1/2) pi / H, phi = (c + 1/2) 2 pi / W - pi,
 * direction (sin theta sin phi, cos theta, -sin theta cos phi): the centre column faces -Z and columns run towards +X.
 * Cube texel (f, r, c) is the fp32 mean of n x n samples, n = dirt_latlong_samples(H, W, S)
 * = max(1, ceil(max(W, 2H) / (pi S))) in float64.  Sample (i, j) lies at sc = (2(c n + j) + 1) / (S n) - 1,
 * tc = (2(r n + i) + 1) / (S n) - 1 on the face's plane (|major| = 1, not normalised); phi = atan2f(x, -z),
 * theta = atan2f(sqrtf(x*x + z*z), y), u = phi * fp32(1/(2 pi)) + 0.5, v = theta * fp32(1/pi), and the bilinear rule of
 * dirt_texture_sample at padded row (v H - 0.5) + 1, column u W - 0.5 of the panorama padded by a copy of row 0 above
 * and of row H-1 below: columns wrap, rows do not.  The n^2 samples are summed in row-major order and the sum divided
 * by n^2, each operation rounded in fp32 in that order.
 * The backward pass writes grad_panorama in full: a gather over the same (sample, texel) pairs in a fixed order, with
 * no atomics and no scratch, so bit-reproducible.
 * H, W in 1 .. 2^20, S in 1 .. 2^14, n <= 4096 (n^2 exact in fp32), else DIRT_ERR_BAD_SHAPE (dirt_latlong_samples
 * returns 0 for H, W or S below 1).  TB = 0: nothing is launched.  All pointers 4-byte aligned; 8- or 16-byte aligned
 * rows enable the vector paths for C = 2, 4. */
int dirt_latlong_samples(int H, int W, int S);
int dirt_latlong_to_cubemap(const float* panorama, float* cubemap, int TB, int H, int W, int S, int C, void* cuda_stream);
int dirt_latlong_to_cubemap_backward(const float* grad_cubemap, float* grad_panorama, int TB, int H, int W, int S, int C,
                                     void* cuda_stream);

/* Reflectance models of the reference's lighting module (dirt/lighting.py:182-343), one value per point and channel.
 * B items of V points each, C channels:
 *   normals, positions   float32 [B*V, 3], row stride normals_stride / positions_stride floats, unit stride along the row
 *   colors               float32 [B*V, C] (vertex colours or reflectivities), row stride colors_stride
 *   light                float32 [B, 3] (light_per_item != 0) or [3] (shared): direction, or position for the point light
 *   light_color          float32 [B, C] or [C];  camera float32 [B, 3] or [3];  shininess float32 [B] or [1]
 *   out, grad_out        float32 [B*V, C], contiguous
 * Per point, with m = -light, term(x) = double_sided ? |x| : max(x, 0), and out_c = (light_color_c * color_c) * f:
 *   DIRT_LIGHT_DIFFUSE_DIRECTIONAL   f = term(n . m)                                  (positions, camera, shininess unused)
 *   DIRT_LIGHT_SPECULAR_DIRECTIONAL  r = light + (2 (n . m)) n,  tc = camera - p,
 *                                    f = pow(term((tc / |tc| + 1e-12) . r), shininess)   (NaN when p == camera)
 *   DIRT_LIGHT_DIFFUSE_POINT         q = p - light,  f = term(n . (q / (|q| + 1e-12)))  (camera, shininess unused)
 * Dot products are fma(a2, b2, fma(a1, b1, a0 * b0)); every other operation is one IEEE-rounded fp32 operation in the
 * order written (pow is powf).
 * Backward: the gradients torch autograd gives for the same expressions (at kinks too: no gradient through |x| at 0,
 * the full gradient through max(x, 0) at 0, none through a zero vector's norm, pow's masks for exponent 0 and base 0).
 * Each gradient output may be NULL, and its work is skipped; the per-point ones are contiguous [B*V, k], the
 * parameter ones have the shape of their input.  Parameter gradients are summed in a fixed order (per-CTA partials in
 * the workspace, then one reduction kernel): repeated calls give bit-identical results.  The workspace, of at least
 * dirt_lighting_workspace_bytes(B, V, C) bytes, is needed only when a parameter gradient is wanted.
 * B = 0 or V = 0: nothing is launched (the backward call still zeroes the wanted parameter gradients).
 * All pointers 4-byte aligned; row strides >= 0. */
enum {
    DIRT_LIGHT_DIFFUSE_DIRECTIONAL = 0,
    DIRT_LIGHT_SPECULAR_DIRECTIONAL = 1,
    DIRT_LIGHT_DIFFUSE_POINT = 2
};
size_t dirt_lighting_workspace_bytes(int B, long long V, int C);
int dirt_lighting_forward(int model, int double_sided,
                          const float* normals, long long normals_stride,
                          const float* positions, long long positions_stride,
                          const float* colors, long long colors_stride,
                          const float* light, int light_per_item, const float* light_color, int light_color_per_item,
                          const float* camera, int camera_per_item, const float* shininess, int shininess_per_item,
                          float* out, int B, long long V, int C, void* cuda_stream);
int dirt_lighting_backward(int model, int double_sided,
                           const float* normals, long long normals_stride,
                           const float* positions, long long positions_stride,
                           const float* colors, long long colors_stride,
                           const float* light, int light_per_item, const float* light_color, int light_color_per_item,
                           const float* camera, int camera_per_item, const float* shininess, int shininess_per_item,
                           const float* grad_out,
                           float* grad_normals, float* grad_positions, float* grad_colors,
                           float* grad_light, float* grad_light_color, float* grad_camera, float* grad_shininess,
                           void* workspace, size_t workspace_bytes, int B, long long V, int C, void* cuda_stream);

/* GGX microfacet specular reflectance (Cook-Torrance with the Trowbridge-Reitz distribution, height-correlated Smith
 * visibility and Schlick's Fresnel term) under one directional (point_light == 0) or point light, one value per point
 * and channel.  B items of V points each, C channels:
 *   normals, positions   float32 [B*V, 3], row stride normals_stride / positions_stride floats, unit stride along the row
 *   roughness            float32 [B*V, 1] (perceptual roughness), row stride roughness_stride
 *   specular             float32 [B*V, C] (the specular colour F0), row stride specular_stride
 *   light                float32 [B, 3] (light_per_item != 0) or [3] (shared): direction, or position (point light)
 *   light_color          float32 [B, C] or [C];  camera float32 [B, 3] or [3]
 *   out, grad_out        float32 [B*V, C], contiguous
 * Per point, with unit(x) = x / (|x| + 1e-12):
 *   n = unit(normal), v = unit(camera - p), l = unit(-light) (directional) or unit(light - p) (point; no falloff)
 *   double_sided and n . v < 0: n = -n
 *   h = unit(l + v), a = max(roughness, 0.045), A = a^4, k = A (n . h)^2 + |n x h|^2, D = A / (pi k^2)
 *   Vis = 0.5 / ((n . l) sqrt((n . v)^2 (1 - A) + A) + (n . v) sqrt((n . l)^2 (1 - A) + A))
 *   F_c = F0_c + (1 - F0_c) (1 - v . h)^5
 *   out_c = pi light_color_c F_c D Vis (n . l) where n . l > 0 and n . v > 0, else 0
 * The geometry and the scalar chain are evaluated in double precision, the channels in fp32; the result is not
 * bit-identical to any torch evaluation.
 * Backward: the gradients torch autograd gives for the same expressions: none where the output is masked to 0, none to
 * a roughness below 0.045 (the full one at exactly 0.045), none through a zero vector's norm.  Each gradient output
 * may be NULL, and its work is skipped; the per-point ones are contiguous [B*V, k], the parameter ones have the shape
 * of their input.  Parameter gradients are summed in a fixed order (per-CTA partials in the workspace, then one
 * reduction kernel): repeated calls give bit-identical results.  The workspace, of at least
 * dirt_lighting_workspace_bytes(B, V, C) bytes, is needed only when a parameter gradient is wanted.
 * B = 0 or V = 0: nothing is launched (the backward call still zeroes the wanted parameter gradients).
 * All pointers 4-byte aligned; row strides >= 0. */
int dirt_ggx_lighting_forward(int point_light, int double_sided,
                              const float* normals, long long normals_stride,
                              const float* positions, long long positions_stride,
                              const float* roughness, long long roughness_stride,
                              const float* specular, long long specular_stride,
                              const float* light, int light_per_item, const float* light_color, int light_color_per_item,
                              const float* camera, int camera_per_item,
                              float* out, int B, long long V, int C, void* cuda_stream);
int dirt_ggx_lighting_backward(int point_light, int double_sided,
                               const float* normals, long long normals_stride,
                               const float* positions, long long positions_stride,
                               const float* roughness, long long roughness_stride,
                               const float* specular, long long specular_stride,
                               const float* light, int light_per_item, const float* light_color, int light_color_per_item,
                               const float* camera, int camera_per_item,
                               const float* grad_out,
                               float* grad_normals, float* grad_positions, float* grad_roughness, float* grad_specular,
                               float* grad_light, float* grad_light_color, float* grad_camera,
                               void* workspace, size_t workspace_bytes, int B, long long V, int C, void* cuda_stream);

/* Spherical-harmonics environment lighting: Lambertian reflected radiance under order-2 SH incident radiance
 * (Ramamoorthi & Hanrahan 2001), one value per point and channel.  B items of V points each, C channels:
 *   normals              float32 [B*V, 3], row stride normals_stride floats, unit stride along the row; used as given
 *                        (not normalised)
 *   albedo               float32 [B*V, C], row stride albedo_stride
 *   coefficients         float32 [B, 9, C] (coefficients_per_item != 0) or [9, C] (shared): L_kc, k = l^2 + l + m
 *   out, grad_out        float32 [B*V, C], contiguous
 * With n = (x, y, z), the real basis without the Condon-Shortley phase
 *   Y0 = 0.28209479177387814, (Y1, Y2, Y3) = 0.4886025119029199 (y, z, x),
 *   (Y4, Y5, Y7) = 1.0925484305920792 (x y, y z, x z), Y6 = 0.31539156525252005 (3 z^2 - 1),
 *   Y8 = 0.5462742152960396 (x^2 - y^2),
 * and the band weights w = 1, 2/3, 1/4 for l = 0, 1, 2:
 *   out_c = albedo_c * E_c,  E_c = sum_{k = 0..8} (w_l(k) L_kc) Y_k, summed in that order with fused multiply-adds;
 *   every other operation is one IEEE-rounded fp32 operation.
 * Backward: the gradients torch autograd gives for the same expressions.  Each gradient output may be NULL, and its work
 * is skipped; grad_normals [B*V, 3] and grad_albedo [B*V, C] are contiguous, grad_coefficients has the shape of
 * coefficients.  The coefficient gradient is summed in a fixed order (per-CTA partials in the workspace, then one
 * reduction kernel, no float atomics): repeated calls give bit-identical results.  The workspace, of at least
 * dirt_sh_lighting_workspace_bytes(B, V, C) bytes (a function of the shapes alone), is needed only when
 * grad_coefficients is wanted.
 * B = 0 or V = 0: nothing is launched (the backward call still zeroes a wanted grad_coefficients).
 * All pointers 4-byte aligned; row strides >= 0; C <= 2^26. */
size_t dirt_sh_lighting_workspace_bytes(int B, long long V, int C);
int dirt_sh_lighting_forward(const float* normals, long long normals_stride,
                             const float* albedo, long long albedo_stride,
                             const float* coefficients, int coefficients_per_item,
                             float* out, int B, long long V, int C, void* cuda_stream);
int dirt_sh_lighting_backward(const float* normals, long long normals_stride,
                              const float* albedo, long long albedo_stride,
                              const float* coefficients, int coefficients_per_item,
                              const float* grad_out,
                              float* grad_normals, float* grad_albedo, float* grad_coefficients,
                              void* workspace, size_t workspace_bytes, int B, long long V, int C, void* cuda_stream);

/* Vertex normals of the reference's lighting module (dirt/lighting.py:34-133) for B items of V vertices sharing the
 * faces:
 *   vertices             float32 [B*V, 3], row stride vertex_stride >= 3 floats, unit stride along the row (the first
 *                        three columns of a [B, V, 4] tensor go in as they are, with vertex_stride 4)
 *   faces                int32 [F, 3], shared by the batch
 *   normals, grad_normals, grad_vertices   float32 [B*V, 3], contiguous
 * With u_f = n_f / (|n_f| + 1e-12), n_f = (p1 - p0) x (p2 - p0) for the corners p0, p1, p2 of face f:
 *   DIRT_NORMALS_AVERAGE    normal_v = s_v / (|s_v| + 1e-12), s_v = sum of u_f over every corner of every face that
 *                           is v (a face naming v twice adds twice)
 *   DIRT_NORMALS_PRE_SPLIT  normal_v = u_f of the last face corner naming v, corner-major then by face (0 if none)
 * A face with an index outside [0, V) is left out: it adds nothing and receives no gradient.
 * Backward: grad_vertices = the gradient torch autograd gives the same expressions (no gradient through the norm of a
 * zero vector; the division by |x| + 1e-12 passes its full 1e12).  Pre-split, grad_normals of v reaches only the face
 * corner whose normal v took, and the positions of every face reach all three of its vertices.
 * Workspace: at least dirt_normals_workspace_bytes(B, V, F) bytes (0 when B, V or F is 0), a function of the sizes
 * alone.  The forward call writes the vertex -> face-corner adjacency into it, and the backward call reads it there:
 * pass the backward call the workspace of the forward call on the same faces and V, with nothing written to it since.
 * The backward call also uses the rest of the workspace as scratch.
 * Every sum has one fixed order (no float atomics): repeated calls give bit-identical normals and gradients.
 * B = 0 or V = 0: nothing is launched; F = 0: the outputs are zeroed.  V < 2^31, 3F < 2^31; all pointers 4-byte
 * aligned. */
enum {
    DIRT_NORMALS_AVERAGE = 0,
    DIRT_NORMALS_PRE_SPLIT = 1
};
size_t dirt_normals_workspace_bytes(int B, long long V, long long F);
int dirt_normals_forward(int mode, const float* vertices, long long vertex_stride, const int32_t* faces,
                         float* normals, void* workspace, size_t workspace_bytes,
                         int B, long long V, long long F, void* cuda_stream);
int dirt_normals_backward(int mode, const float* vertices, long long vertex_stride, const int32_t* faces,
                          const float* grad_normals, float* grad_vertices, void* workspace, size_t workspace_bytes,
                          int B, long long V, long long F, void* cuda_stream);

/* Vertex tangents for tangent-space normal mapping, for B items of V vertices sharing the faces:
 *   vertices             float32 [B*V, 3], row stride vertex_stride >= 3 floats, unit stride along the row
 *   uvs                  float32, the uv of vertex v of item b at uvs + b*uv_item_stride + v*uv_stride, uv_stride >= 2,
 *                        unit stride along the row (uv_item_stride 0: one set shared by the batch)
 *   normals              float32 [B*V, 3], row stride normals_stride >= 3, e.g. the output of dirt_normals_forward
 *   faces                int32 [F, 3], shared by the batch
 *   tangents, grad_tangents   float32 [B*V, 4], contiguous
 * With unit(x) = x / (|x| + 1e-12) and, for face f with corners p0, p1, p2 and uvs (u_k, v_k),
 * e1 = p1 - p0, e2 = p2 - p0, (du_k, dv_k) = uv_k - uv0, s = sign(du1 dv2 - du2 dv1) (0 when it is 0):
 *   t_f = unit(s (e1 dv2 - e2 dv1)),  b_f = unit(s (e2 du1 - e1 du2)),
 *   t_v, b_v = the sums of t_f, b_f over every corner of every face that is v,  n = unit(normal_v),
 *   tangent_v = (T, w),  T = unit(t_v - (n . t_v) n),  w = -1 if (n x T) . b_v < 0 else +1.
 * A face with degenerate uvs adds nothing; a vertex no face names gets (0, 0, 0, 1).  A face with an index outside
 * [0, V) is left out.
 * Backward: the gradients torch autograd gives the same expressions.  None passes through w or the sign, so du gets 0;
 * the w column of grad_tangents is ignored.  grad_vertices [B*V, 3], grad_uvs [B*V, 2] (one row per item and vertex,
 * also for shared uvs: the caller sums them over the items) and grad_normals [B*V, 3] are contiguous; each may be NULL,
 * and its work is skipped.
 * Workspace: dirt_tangents_workspace_bytes(B, V, F) bytes, the layout of dirt_normals_workspace_bytes.  The forward
 * call writes the vertex -> face-corner adjacency into it and the backward call reads it there, as for the normals.
 * Every sum has one fixed order (no float atomics): repeated calls give bit-identical tangents and gradients.
 * B = 0 or V = 0: nothing is launched; F = 0: every vertex gets (0, 0, 0, 1) and the gradients are zeroed.
 * V < 2^31, 3F < 2^31; all pointers 4-byte aligned. */
size_t dirt_tangents_workspace_bytes(int B, long long V, long long F);
int dirt_tangents_forward(const float* vertices, long long vertex_stride, const float* uvs, long long uv_stride,
                          long long uv_item_stride, const float* normals, long long normals_stride, const int32_t* faces,
                          float* tangents, void* workspace, size_t workspace_bytes,
                          int B, long long V, long long F, void* cuda_stream);
int dirt_tangents_backward(const float* vertices, long long vertex_stride, const float* uvs, long long uv_stride,
                           long long uv_item_stride, const float* normals, long long normals_stride, const int32_t* faces,
                           const float* grad_tangents, float* grad_vertices, float* grad_uvs, float* grad_normals,
                           void* workspace, size_t workspace_bytes, int B, long long V, long long F, void* cuda_stream);

/* Tangent-space normal mapping, one value per point.  B items of V points each:
 *   normals              float32 [B*V, 3], row stride normals_stride (interpolated: not unit length)
 *   tangents             float32 [B*V, 4], row stride tangents_stride (interpolated dirt_tangents_forward output)
 *   samples              float32 [B*V, 3], row stride samples_stride: the tangent-space normal, decoded to [-1, 1]
 *   out, grad_out        float32 [B*V, 3], contiguous
 * With unit(x) = x / (|x| + 1e-12), n = unit(normal), T = unit(t.xyz - (n . t.xyz) n), s = -1 if t.w < 0 else +1:
 *   out = unit(m.x T + m.y s (n x T) + m.z n);  a point with n = 0 gives 0.
 * Backward: the gradients torch autograd gives the same expressions.  grad_normals [B*V, 3], grad_tangents [B*V, 4]
 * (its w column 0) and grad_samples [B*V, 3] are contiguous; each may be NULL, and its work is skipped.
 * B = 0 or V = 0: nothing is launched.  All pointers 4-byte aligned; row strides >= 0. */
int dirt_normal_map_forward(const float* normals, long long normals_stride, const float* tangents,
                            long long tangents_stride, const float* samples, long long samples_stride,
                            float* out, int B, long long V, void* cuda_stream);
int dirt_normal_map_backward(const float* normals, long long normals_stride, const float* tangents,
                             long long tangents_stride, const float* samples, long long samples_stride,
                             const float* grad_out, float* grad_normals, float* grad_tangents, float* grad_samples,
                             int B, long long V, void* cuda_stream);

/* Shadow-map visibility: a percentage-closer lookup of a light-view map, one value per point.  B items of V points:
 *   positions            float32 [B*V, 3] world points, row stride positions_stride, unit stride along the row
 *   light_matrix         float32 [B, 4, 4] (per_item) or [4, 4]: world -> light clip, row vectors ((p, 1) @ M)
 *   shadow_map           float32 [B, SH, SW, 2] (per_item) or [SH, SW, 2], contiguous and 8-byte aligned: per texel
 *                        (occupancy, depth), e.g. a rasterisation from the light with vertex colours (1, clip z)
 *   out, grad_out        float32 [B*V], contiguous
 * With (x, y, z, w) = (p, 1) @ M, X = (x/w + 1) (0.5 SW) and Yd = (1 - y/w) (0.5 SH) (the rasteriser's pixel rule;
 * this chain is evaluated in double precision), u = X - 0.5, c0 = floor(u), fc = u - c0, and r0, fr the same of
 * Yd - 0.5:
 *   out = sum_i sum_k a_i b_k s_ik / (2R+1)^2 over rows r0-R+i and columns c0-R+k, i, k = 0 .. 2R+1, each clamped into
 *   the map; a = (1 - fr, 1, ..., 1, fr), b = (1 - fc, 1, ..., 1, fc);
 *   s_ik = 1 - o_ik step((z - z_ik - bias) / softness), step the logistic sigmoid for softness > 0, and for
 *   softness = 0 the Heaviside step with step(0) = 0.
 * A non-finite (x, y, z, w), w <= 0, or (X, Yd) outside [0, SW) x [0, SH) gives out = 1 and no gradient.
 * Backward: the gradients torch autograd gives the same expressions (none through the step for softness = 0).
 * grad_positions [B*V, 3] is contiguous, grad_light_matrix and grad_shadow_map (8-byte aligned) have the shapes of
 * their inputs; each may be NULL, and its work is skipped.  The light-matrix gradient is summed in a fixed order
 * (per-CTA partials in the workspace, of at least dirt_shadow_workspace_bytes(B, V) bytes, needed only when it is
 * wanted), so repeated calls give bit-identical results.  The map gradient is summed with float atomics after
 * aggregation inside each warp: its last bits may differ between calls (see dirt_shadow_backward_deterministic).
 * B = 0 or V = 0: nothing is launched (the backward call still zeroes wanted map and matrix gradients).
 * 0 <= radius <= 3, softness and bias finite and >= 0, SH, SW > 0; all pointers 4-byte aligned; row stride >= 0.
 * dirt_shadow_backward_deterministic: the same gradients with the map gradient summed without float atomics, so that
 * repeated calls give bit-identical results.  The points are sorted by base texel (r0, c0), and each texel sums, in
 * float64 from +0.0 and rounded once, the backward call's fp32 terms in this order: tap row i, the base rows whose tap
 * row i clamps onto it (ascending), tap column k, the base columns likewise, then the points of that base in ascending
 * id b*V + n (DESIGN.md §7.15).  Its scratch, of at least dirt_shadow_backward_deterministic_bytes(B, V, per_item, SH,
 * SW) bytes, is needed only when grad_shadow_map is wanted; B*V and (B | 1)(SH + 1)(SW + 1) below 2^31. */
size_t dirt_shadow_workspace_bytes(int B, long long V);
size_t dirt_shadow_backward_deterministic_bytes(int B, long long V, int per_item, int SH, int SW);
int dirt_shadow_forward(const float* positions, long long positions_stride, const float* light_matrix,
                        const float* shadow_map, int per_item, int SH, int SW, int radius, float softness, float bias,
                        float* out, int B, long long V, void* cuda_stream);
int dirt_shadow_backward(const float* positions, long long positions_stride, const float* light_matrix,
                         const float* shadow_map, int per_item, int SH, int SW, int radius, float softness, float bias,
                         const float* grad_out, float* grad_positions, float* grad_light_matrix, float* grad_shadow_map,
                         void* workspace, size_t workspace_bytes, int B, long long V, void* cuda_stream);
int dirt_shadow_backward_deterministic(const float* positions, long long positions_stride, const float* light_matrix,
                                       const float* shadow_map, int per_item, int SH, int SW, int radius,
                                       float softness, float bias, const float* grad_out, float* grad_positions,
                                       float* grad_light_matrix, float* grad_shadow_map, void* workspace,
                                       size_t workspace_bytes, void* scratch, size_t scratch_bytes, int B, long long V,
                                       void* cuda_stream);

/* Number of kernels the last launching call on this thread launched successfully (bench.py's gpu_launches).  A
 * launch that fails is not counted; the call then returns DIRT_ERR_CUDA.  The size queries, the kernel-timer hooks and
 * dirt_peer_exchange leave the count as it was. */
int dirt_last_launch_count(void);

/* Profiling hooks (replace the reference's compile-time TIME_SECTIONS stamps,
 * csrc/rasterise_egl.cpp:284-286,398-405): bracket ONE kernel of subsequent calls on this thread with
 * CUDA events recorded on the call's own stream.  which: 0 = off, 1 = forward raster kernel,
 * 2 = backward (assemble-grads) kernel, 3 = triangle-setup kernel (of every call that runs it; a
 * backward call handed the forward's workspace does not).  dirt_kernel_timer_elapsed_ms() waits for the last bracketed
 * launch and returns its duration in milliseconds (negative if nothing was timed). */
int dirt_kernel_timer_enable(int which);
float dirt_kernel_timer_elapsed_ms(void);

#ifdef __cplusplus
}
#endif
#endif /* DIRT_B200_H */
