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

/* Number of kernels the last call on this thread launched (bench.py's gpu_launches). */
int dirt_last_launch_count(void);

/* Profiling hooks (replace the reference's compile-time TIME_SECTIONS stamps,
 * csrc/rasterise_egl.cpp:284-286,398-405): bracket ONE kernel of subsequent calls on this thread with
 * CUDA events recorded on the call's own stream.  which: 0 = off, 1 = forward raster kernel,
 * 2 = backward (assemble-grads) kernel.  dirt_kernel_timer_elapsed_ms() waits for the last bracketed
 * launch and returns its duration in milliseconds (negative if nothing was timed). */
int dirt_kernel_timer_enable(int which);
float dirt_kernel_timer_elapsed_ms(void);

#ifdef __cplusplus
}
#endif
#endif /* DIRT_B200_H */
