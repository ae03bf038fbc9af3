// api.cu -- the C ABI of libdirt_b200.so (include/dirt_b200.h): argument validation, workspace
// carving and kernel sequencing.  No device allocation, no host synchronisation, no global state
// other than a thread-local launch counter.
#include "../../include/dirt_b200.h"
#include "common.cuh"

#include <cmath>
#include <initializer_list>

using namespace dirt;

static_assert(BWD_SHARED_GEOMETRY == DIRT_BWD_SHARED_GEOMETRY && BWD_SKIP_POSITION == DIRT_BWD_SKIP_POSITION &&
              BWD_SKIP_COLOUR == DIRT_BWD_SKIP_COLOUR, "flag values of common.cuh and dirt_b200.h differ");

extern "C" const char* dirt_error_string(int code)
{
    switch (code) {
        case DIRT_OK: return "ok";
        case DIRT_ERR_BAD_SHAPE:
            return "bad shape: need B >= 0, H > 0, W > 0, C > 0, V >= 0, F >= 0 (and sizes within int32 range)";
        case DIRT_ERR_NULL_POINTER: return "a required pointer is NULL";
        case DIRT_ERR_WORKSPACE_TOO_SMALL: return "workspace smaller than dirt_workspace_bytes()";
        case DIRT_ERR_BAD_CHANNEL_GROUPS: return "channel groups must each be 1 or 3 wide and sum to C";
        case DIRT_ERR_TOO_MANY_VERTICES: return "RasteriseGrad supports a maximum of 16777216 vertices";
        case DIRT_ERR_CUDA: return "a CUDA call or kernel launch failed";
        case DIRT_ERR_MISALIGNED: return "pointer not sufficiently aligned (workspace 256 B, vertices 16 B, others 4 B)";
        case DIRT_ERR_STALE_WORKSPACE:
            return "workspace_holds_setup was set, but the workspace does not hold the setup records of these (vertices, faces, sizes)";
        default: return "unknown error code";
    }
}

extern "C" int dirt_abi_version(void) { return 4; }

namespace dirt {
KernelTimer& kernel_timer()
{
    static thread_local KernelTimer t;
    return t;
}

int& launch_count()
{
    static thread_local int n = 0;
    return n;
}
}  // namespace dirt

extern "C" int dirt_kernel_timer_enable(int which)
{
    KernelTimer& t = kernel_timer();
    if (which < 0 || which > 3) return DIRT_ERR_BAD_SHAPE;
    if (which != 0 && !t.start) {
        if (cudaEventCreate(&t.start) != cudaSuccess || cudaEventCreate(&t.stop) != cudaSuccess) {
            t.start = t.stop = nullptr;
            return DIRT_ERR_CUDA;
        }
    }
    t.which = which;
    t.recorded = false;
    return DIRT_OK;
}

extern "C" float dirt_kernel_timer_elapsed_ms(void)
{
    KernelTimer& t = kernel_timer();
    if (!t.recorded) return -1.f;
    float ms = -1.f;
    if (cudaEventSynchronize(t.stop) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, t.start, t.stop) != cudaSuccess) return -1.f;
    return ms;
}

extern "C" int dirt_last_launch_count(void) { return launch_count(); }

// gradient outputs may be NULL (not wanted), but not misaligned
static bool aligned(std::initializer_list<const void*> ptrs)
{
    for (const void* p : ptrs)
        if ((uintptr_t)p % 4) return false;
    return true;
}

// buffers a call reads or writes: DIRT_ERR_NULL_POINTER if one is NULL, else DIRT_ERR_MISALIGNED if one is not 4-byte
// aligned
static int required_check(std::initializer_list<const void*> ptrs)
{
    for (const void* p : ptrs)
        if (!p) return DIRT_ERR_NULL_POINTER;
    return aligned(ptrs) ? DIRT_OK : DIRT_ERR_MISALIGNED;
}

// a caller-owned workspace or scratch of `bytes` bytes that a call needs `need` of: DIRT_ERR_NULL_POINTER if it is NULL,
// else DIRT_ERR_MISALIGNED if it is not 256-byte aligned, else DIRT_ERR_WORKSPACE_TOO_SMALL if it is too small
static int scratch_check(const void* scratch, size_t bytes, size_t need)
{
    if (!scratch) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)scratch % 256) return DIRT_ERR_MISALIGNED;
    return bytes < need ? DIRT_ERR_WORKSPACE_TOO_SMALL : DIRT_OK;
}

static bool shape_ok(int B, int H, int W, int C, int V, int F)
{
    if (B < 0 || H <= 0 || W <= 0 || C <= 0 || V < 0 || F < 0) return false;
    if (C / 3 + C % 3 > MAX_GROUPS) return false;             // the greedy split of C (groups of 3, then of 1) must fit GroupSpec
    if ((long long)H * W > (1ll << 30)) return false;         // row*W+col stays in int32
    if ((long long)W > (1 << 18) || (long long)H > (1 << 18)) return false;
    if ((long long)B * F > (1ll << 31) - 1) return false;
    if ((long long)B * ((W + TILE_W - 1) / TILE_W) * ((H + TILE_H - 1) / TILE_H) > (1ll << 31) - 1) return false;   // tile indices are int32
    return true;
}

extern "C" size_t dirt_workspace_bytes(int B, int H, int W, int C, int V, int F)
{
    if (!shape_ok(B, H, W, C > 0 ? C : 1, V, F)) return 0;
    Workspace ws = carve_workspace(nullptr, B, H, W, C, V, F);
    return ws.bytes + 256;
}

static int make_groups(int C, const int* channel_groups, int n_groups, GroupSpec* g)
{
    g->n = 0;
    if (channel_groups && n_groups > 0) {
        if (n_groups > MAX_GROUPS) return DIRT_ERR_BAD_CHANNEL_GROUPS;
        int sum = 0;
        for (int i = 0; i < n_groups; ++i) {
            if (channel_groups[i] != 1 && channel_groups[i] != 3) return DIRT_ERR_BAD_CHANNEL_GROUPS;
            g->width[i] = (unsigned char)channel_groups[i];
            sum += channel_groups[i];
        }
        if (sum != C) return DIRT_ERR_BAD_CHANNEL_GROUPS;
        g->n = n_groups;
        return DIRT_OK;
    }
    // the reference's own greedy split (dirt/rasterise_ops.py:80-108)
    if (C == 1 || C == 3) { g->width[0] = (unsigned char)C; g->n = 1; return DIRT_OK; }
    int begin = 0;
    while (begin < C) {
        const int w = (begin + 3 <= C) ? 3 : 1;
        if (g->n >= MAX_GROUPS) return DIRT_ERR_BAD_CHANNEL_GROUPS;
        g->width[g->n++] = (unsigned char)w;
        begin += w;
    }
    return DIRT_OK;
}

extern "C" size_t dirt_workspace_bytes_min(int B, int H, int W, int C, int V, int F)
{
    if (!shape_ok(B, H, W, C > 0 ? C : 1, V, F)) return 0;
    Workspace ws = carve_workspace(nullptr, B, H, W, C, V, F);
    return ws.bytes_without_face_ids + 256;
}

#define CUDA_TRY(expr)                                   \
    do {                                                 \
        if ((expr) != cudaSuccess) return DIRT_ERR_CUDA; \
    } while (0)

// The checks the rasteriser entries share, in order: NULL (DIRT_ERR_NULL_POINTER) for `required`, for `per_vertex` when
// V > 0 and for `faces` when F > 0; 16-byte alignment of `aligned16`, then 4-byte alignment of `aligned4`
// (DIRT_ERR_MISALIGNED); the workspace against `need`.  Before it each entry makes its shape check, its own checks
// (backward: vertex limit, flags, channel groups; derivatives: channel range) and its DIRT_OK return for B == 0.
// What stays per entry:
// - visibility NULL-checks only vertices and faces, and aligns its face ids but not the faces; its G-buffer may be NULL;
// - backward first requires pixels unless DIRT_BWD_SKIP_POSITION and grad_background unless DIRT_BWD_SKIP_COLOUR; without
//   face ids it needs dirt_workspace_bytes (room to derive them), and the deterministic entry then checks its scratch.
static int raster_check(int V, int F, const int32_t* faces, std::initializer_list<const void*> required,
                        std::initializer_list<const void*> per_vertex, std::initializer_list<const void*> aligned16,
                        std::initializer_list<const void*> aligned4, const void* workspace, size_t bytes, size_t need)
{
    for (const void* p : required)
        if (!p) return DIRT_ERR_NULL_POINTER;
    for (const void* p : per_vertex)
        if (V > 0 && !p) return DIRT_ERR_NULL_POINTER;
    if (F > 0 && !faces) return DIRT_ERR_NULL_POINTER;
    for (const void* p : aligned16)
        if ((uintptr_t)p % 16) return DIRT_ERR_MISALIGNED;
    return aligned(aligned4) ? scratch_check(workspace, bytes, need) : DIRT_ERR_MISALIGNED;
}

// the workspace blocks, launch sizes and stream of one rasteriser call
struct RasterCall { Workspace ws; Dims d; cudaStream_t stream; };

static RasterCall raster_call(const void* workspace, int B, int H, int W, int C, int V, int F, void* cuda_stream)
{
    return {carve_workspace(const_cast<void*>(workspace), B, H, W, C, V, F), make_dims(B, H, W, C, V, F),
            (cudaStream_t)cuda_stream};
}

extern "C" int dirt_rasterise_forward(const float* background, const float* vertices, const float* vertex_colors,
                                      const int32_t* faces, float* pixels, int32_t* face_ids_out, int B, int H, int W,
                                      int C, int V, int F, void* workspace, size_t workspace_bytes, void* cuda_stream)
{
    launch_count() = 0;
    if (!shape_ok(B, H, W, C, V, F)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0) return DIRT_OK;
    const int rc = raster_check(V, F, faces, {background, pixels}, {vertices, vertex_colors}, {vertices},
                                {background, pixels, vertex_colors, faces, face_ids_out}, workspace, workspace_bytes,
                                dirt_workspace_bytes_min(B, H, W, C, V, F));
    if (rc != DIRT_OK) return rc;
    const RasterCall r = raster_call(workspace, B, H, W, C, V, F, cuda_stream);
    CUDA_TRY(launch_setup_and_bin(vertices, faces, vertex_colors, r.ws, r.d, r.stream));
#if !defined(DIRT_SETUP_ABLATE) || DIRT_SETUP_ABLATE == 0   // a setup timing build leaves the records undefined
    CUDA_TRY(launch_raster_forward(vertices, background, vertex_colors, pixels, face_ids_out, r.ws, r.d, r.stream));
#endif
    return DIRT_OK;
}

extern "C" int dirt_rasterise_visibility(const float* vertices, const int32_t* faces, int32_t* face_ids, float* gbuffer,
                                         int B, int H, int W, int V, int F, void* workspace, size_t workspace_bytes,
                                         void* cuda_stream)
{
    launch_count() = 0;
    if (!shape_ok(B, H, W, 1, V, F)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0) return DIRT_OK;
    const int rc = raster_check(V, F, faces, {}, {vertices}, {vertices, gbuffer}, {face_ids}, workspace, workspace_bytes,
                                dirt_workspace_bytes_min(B, H, W, 1, V, F));
    if (rc != DIRT_OK) return rc;
    const RasterCall r = raster_call(workspace, B, H, W, 1, V, F, cuda_stream);
    CUDA_TRY(launch_setup_and_bin(vertices, faces, nullptr, r.ws, r.d, r.stream));
    CUDA_TRY(launch_raster_visibility(vertices, face_ids, gbuffer, r.ws, r.d, r.stream));
    return DIRT_OK;
}

// The three backward entries.  The deterministic one adds its int32 rule (the adjacency's corner ids b*3F + k*F + f, a
// second DIRT_ERR_BAD_SHAPE check) and its scratch.
static int backward_impl(const float* vertices, const int32_t* faces, const float* pixels, const float* grad_pixels,
                         const int32_t* face_ids, float* grad_background, float* grad_vertices, float* grad_vertex_colors,
                         int B, int H, int W, int C, int V, int F, const int* channel_groups, int n_groups,
                         int workspace_holds_setup, int flags, void* workspace, size_t workspace_bytes, void* cuda_stream,
                         bool deterministic = false, void* scratch = nullptr, size_t scratch_bytes = 0)
{
    launch_count() = 0;
    if (!shape_ok(B, H, W, C, V, F) || (deterministic && 3ll * B * F > (1ll << 31) - 1)) return DIRT_ERR_BAD_SHAPE;
    if (V > (1 << 24)) return DIRT_ERR_TOO_MANY_VERTICES;
    if (flags & ~(DIRT_BWD_SHARED_GEOMETRY | DIRT_BWD_SKIP_POSITION | DIRT_BWD_SKIP_COLOUR)) return DIRT_ERR_BAD_SHAPE;
    GroupSpec groups;
    int rc = make_groups(C, channel_groups, n_groups, &groups);
    if (rc != DIRT_OK) return rc;
    if (B == 0) return DIRT_OK;
    if ((!(flags & DIRT_BWD_SKIP_POSITION) && !pixels) || (!(flags & DIRT_BWD_SKIP_COLOUR) && !grad_background))
        return DIRT_ERR_NULL_POINTER;
    rc = raster_check(V, F, faces, {grad_pixels}, {vertices, grad_vertices, grad_vertex_colors}, {vertices, grad_vertices},
                      {pixels, grad_pixels, grad_background, grad_vertex_colors, faces, face_ids}, workspace, workspace_bytes,
                      face_ids ? dirt_workspace_bytes_min(B, H, W, C, V, F) : dirt_workspace_bytes(B, H, W, C, V, F));
    if (rc == DIRT_OK && deterministic)
        rc = scratch_check(scratch, scratch_bytes, dirt_rasterise_backward_deterministic_bytes(B, H, W, C, V, F));
    if (rc != DIRT_OK) return rc;
    const RasterCall r = raster_call(workspace, B, H, W, C, V, F, cuda_stream);
    const int32_t* ids = face_ids;
    // the tile coverage flags in the workspace describe `ids` when the raster kernel that produced them ran on this workspace
    const bool flags_valid = !ids || workspace_holds_setup;
    unsigned long long expect_tag = 0;
    if (!ids) {
        // no cached visibility: re-derive it exactly as the forward pass does
        CUDA_TRY(launch_setup_and_bin(vertices, faces, nullptr, r.ws, r.d, r.stream));
        CUDA_TRY(launch_raster_visibility(vertices, r.ws.face_ids, nullptr, r.ws, r.d, r.stream));
        ids = r.ws.face_ids;
    } else if (!workspace_holds_setup) {
        CUDA_TRY(launch_setup_only(vertices, faces, r.ws, r.d, r.stream));
    } else {
        // a promise: checked on the device against the tag the setup pass left in the workspace
        expect_tag = workspace_tag(vertices, faces, B, H, W, V, F);
    }
    if (deterministic)
        CUDA_TRY(launch_backward_deterministic(vertices, faces, pixels, grad_pixels, ids, grad_background, grad_vertices,
                                               grad_vertex_colors, r.ws, r.d, groups, flags, expect_tag,
                                               carve_det_scratch(scratch, B, H, W, C, V, F), r.stream));
    else
        CUDA_TRY(launch_backward(vertices, pixels, grad_pixels, ids, grad_background, grad_vertices, grad_vertex_colors, r.ws,
                                 r.d, groups, flags_valid, flags, expect_tag, r.stream));
    return DIRT_OK;
}

extern "C" int dirt_rasterise_backward(const float* vertices, const int32_t* faces, const float* pixels,
                                       const float* grad_pixels, const int32_t* face_ids, float* grad_background,
                                       float* grad_vertices, float* grad_vertex_colors, int B, int H, int W, int C, int V,
                                       int F, const int* channel_groups, int n_groups, int workspace_holds_setup,
                                       void* workspace, size_t workspace_bytes, void* cuda_stream)
{
    return backward_impl(vertices, faces, pixels, grad_pixels, face_ids, grad_background, grad_vertices, grad_vertex_colors, B, H,
                         W, C, V, F, channel_groups, n_groups, workspace_holds_setup, 0, workspace, workspace_bytes, cuda_stream);
}

extern "C" int dirt_rasterise_backward_ex(const float* vertices, const int32_t* faces, const float* pixels,
                                          const float* grad_pixels, const int32_t* face_ids, float* grad_background,
                                          float* grad_vertices, float* grad_vertex_colors, int B, int H, int W, int C, int V,
                                          int F, const int* channel_groups, int n_groups, int workspace_holds_setup, int flags,
                                          void* workspace, size_t workspace_bytes, void* cuda_stream)
{
    return backward_impl(vertices, faces, pixels, grad_pixels, face_ids, grad_background, grad_vertices, grad_vertex_colors, B, H,
                         W, C, V, F, channel_groups, n_groups, workspace_holds_setup, flags, workspace, workspace_bytes, cuda_stream);
}

extern "C" size_t dirt_rasterise_backward_deterministic_bytes(int B, int H, int W, int C, int V, int F)
{
    if (!shape_ok(B, H, W, C > 0 ? C : 1, V, F) || B == 0) return 0;
    return carve_det_scratch(nullptr, B, H, W, C, V, F).bytes;
}

extern "C" int dirt_rasterise_backward_deterministic(const float* vertices, const int32_t* faces, const float* pixels,
                                                     const float* grad_pixels, const int32_t* face_ids, float* grad_background,
                                                     float* grad_vertices, float* grad_vertex_colors, int B, int H, int W,
                                                     int C, int V, int F, const int* channel_groups, int n_groups,
                                                     int workspace_holds_setup, int flags, void* workspace,
                                                     size_t workspace_bytes, void* scratch, size_t scratch_bytes,
                                                     void* cuda_stream)
{
    return backward_impl(vertices, faces, pixels, grad_pixels, face_ids, grad_background, grad_vertices, grad_vertex_colors, B, H,
                         W, C, V, F, channel_groups, n_groups, workspace_holds_setup, flags, workspace, workspace_bytes,
                         cuda_stream, true, scratch, scratch_bytes);
}

extern "C" int dirt_rasterise_derivatives(const float* vertices, const int32_t* faces, const float* attributes,
                                          const int32_t* face_ids, float* derivatives, int B, int H, int W, int C, int V,
                                          int F, int first_channel, int channel_count, int workspace_holds_setup,
                                          void* workspace, size_t workspace_bytes, void* cuda_stream)
{
    launch_count() = 0;
    if (!shape_ok(B, H, W, C, V, F)) return DIRT_ERR_BAD_SHAPE;
    if (first_channel < 0 || channel_count <= 0 || first_channel >= C || channel_count > C - first_channel)
        return DIRT_ERR_BAD_SHAPE;
    if (B == 0) return DIRT_OK;
    const int rc = raster_check(V, F, faces, {face_ids, derivatives}, {vertices, attributes}, {vertices},
                                {attributes, faces, face_ids, derivatives}, workspace, workspace_bytes,
                                dirt_workspace_bytes_min(B, H, W, C, V, F));
    if (rc != DIRT_OK) return rc;
    const RasterCall r = raster_call(workspace, B, H, W, C, V, F, cuda_stream);
    unsigned long long expect_tag = 0;
    if (!workspace_holds_setup)
        CUDA_TRY(launch_setup_only(vertices, faces, r.ws, r.d, r.stream));
    else
        expect_tag = workspace_tag(vertices, faces, B, H, W, V, F);   // checked on the device, as backward_impl does
    CUDA_TRY(launch_gbuffer_derivatives(face_ids, attributes, derivatives, r.ws, r.d, first_channel, channel_count, expect_tag,
                                        r.stream));
    return DIRT_OK;
}

// texel indices (and the warp keys built from them) stay below 2^62, element offsets of every buffer below 2^62
static bool texture_shape_ok(int TB, int TH, int TW, int C, int B, long long N, int mode)
{
    if (B < 0 || N < 0 || TH <= 0 || TW <= 0 || C <= 0) return false;
    if (TB != 1 && TB != B) return false;
    if (mode != DIRT_TEXTURE_BILINEAR && mode != DIRT_TEXTURE_NEAREST) return false;
    const double limit = 4.0e18;
    if ((double)TB * TH * TW * C > limit || (double)B * N * (C > 2 ? C : 2) > limit) return false;
    return true;
}

static TexDims make_tex_dims(int TB, int TH, int TW, int C, int B, long long N, int mode)
{
    TexDims d;
    d.total = (long long)B * N; d.N = N; d.texels = (long long)TH * TW;
    d.TB = TB; d.TH = TH; d.TW = TW; d.C = C; d.mode = mode;
    return d;
}

extern "C" int dirt_texture_sample(const float* texture, const float* indices, float* out, int TB, int TH, int TW, int C,
                                   int B, long long N, int mode, void* cuda_stream)
{
    launch_count() = 0;
    if (!texture_shape_ok(TB, TH, TW, C, B, N, mode)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0 || N == 0) return DIRT_OK;
    const int rc = required_check({texture, indices, out});
    if (rc != DIRT_OK) return rc;
    CUDA_TRY(launch_texture_forward(texture, indices, out, make_tex_dims(TB, TH, TW, C, B, N, mode), (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_texture_sample_backward(const float* texture, const float* indices, const float* grad_out,
                                            float* grad_texture, float* grad_indices, int TB, int TH, int TW, int C, int B,
                                            long long N, int mode, void* cuda_stream)
{
    launch_count() = 0;
    if (!texture_shape_ok(TB, TH, TW, C, B, N, mode)) return DIRT_ERR_BAD_SHAPE;
    const TexDims d = make_tex_dims(TB, TH, TW, C, B, N, mode);
    if (d.total > 0) {
        if (!indices || !grad_out) return DIRT_ERR_NULL_POINTER;
        if (grad_indices && mode == DIRT_TEXTURE_BILINEAR && !texture) return DIRT_ERR_NULL_POINTER;
    }
    if (!aligned({texture, indices, grad_out, grad_texture, grad_indices})) return DIRT_ERR_MISALIGNED;
    // with no lookups only the memset of grad_texture is enqueued
    CUDA_TRY(launch_texture_backward(texture, indices, grad_out, grad_texture, grad_indices, d, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// the deterministic path's lookup ids and sort keys (texel ids plus one sentinel) are 32-bit
static bool texture_det_shape_ok(int TB, int TH, int TW, int C, int B, long long N, int mode)
{
    return texture_shape_ok(TB, TH, TW, C, B, N, mode) && (long long)B * N < (1ll << 31) &&
           (long long)TB * TH * TW < (1ll << 31) - 1;
}

extern "C" size_t dirt_texture_sample_backward_deterministic_bytes(int TB, int TH, int TW, int C, int B, long long N, int mode)
{
    if (!texture_det_shape_ok(TB, TH, TW, C, B, N, mode) || (long long)B * N == 0) return 0;
    return carve_texture_det_scratch(nullptr, make_tex_dims(TB, TH, TW, C, B, N, mode)).bytes;
}

extern "C" int dirt_texture_sample_backward_deterministic(const float* texture, const float* indices, const float* grad_out,
                                                          float* grad_texture, float* grad_indices, int TB, int TH, int TW,
                                                          int C, int B, long long N, int mode, void* scratch,
                                                          size_t scratch_bytes, void* cuda_stream)
{
    launch_count() = 0;
    if (!texture_det_shape_ok(TB, TH, TW, C, B, N, mode)) return DIRT_ERR_BAD_SHAPE;
    const TexDims d = make_tex_dims(TB, TH, TW, C, B, N, mode);
    if (d.total > 0) {
        if (!indices || !grad_out) return DIRT_ERR_NULL_POINTER;
        if (grad_indices && mode == DIRT_TEXTURE_BILINEAR && !texture) return DIRT_ERR_NULL_POINTER;
    }
    if (!aligned({texture, indices, grad_out, grad_texture, grad_indices})) return DIRT_ERR_MISALIGNED;
    // only the texture gradient of a call with lookups sorts them
    const bool sorts = grad_texture && d.total > 0;
    if (sorts) {
        const int rc = scratch_check(scratch, scratch_bytes,
                                     dirt_texture_sample_backward_deterministic_bytes(TB, TH, TW, C, B, N, mode));
        if (rc != DIRT_OK) return rc;
    }
    CUDA_TRY(launch_texture_backward_deterministic(texture, indices, grad_out, grad_texture, grad_indices, d,
                                                   carve_texture_det_scratch(sorts ? scratch : nullptr, d),
                                                   (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// ---- mipmapped (trilinear) lookup ----

// the bilinear lookup's limits, and the derivatives' 4 floats per lookup
static bool mip_shape_ok(int TB, int TH, int TW, int C, int B, long long N)
{
    return texture_shape_ok(TB, TH, TW, C, B, N, DIRT_TEXTURE_BILINEAR) && (double)B * N * (C > 4 ? C : 4) <= 4.0e18;
}

extern "C" int dirt_texture_mip_levels(int TH, int TW) { return TH > 0 && TW > 0 ? mip_levels(TH, TW) : 0; }

extern "C" size_t dirt_texture_mip_pyramid_bytes(int TB, int TH, int TW, int C)
{
    if (TB < 0 || !texture_shape_ok(TB, TH, TW, C, TB, 0, DIRT_TEXTURE_BILINEAR)) return 0;
    const TexDims d = make_tex_dims(TB, TH, TW, C, TB, 0, DIRT_TEXTURE_BILINEAR);
    return sizeof(float) * (size_t)mip_pyramid_texels(d, mip_levels(TH, TW)) * C;
}

extern "C" int dirt_texture_mip_build(const float* texture, float* pyramid, int TB, int TH, int TW, int C, void* cuda_stream)
{
    launch_count() = 0;
    if (TB < 0 || !texture_shape_ok(TB, TH, TW, C, TB, 0, DIRT_TEXTURE_BILINEAR)) return DIRT_ERR_BAD_SHAPE;
    if (TB == 0 || mip_levels(TH, TW) == 1) return DIRT_OK;
    const int rc = required_check({texture, pyramid});
    if (rc != DIRT_OK) return rc;
    CUDA_TRY(launch_texture_mip_build(texture, pyramid, make_tex_dims(TB, TH, TW, C, TB, 0, DIRT_TEXTURE_BILINEAR),
                                      (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_texture_sample_trilinear(const float* texture, const float* pyramid, const float* indices,
                                             const float* derivatives, float* out, int TB, int TH, int TW, int C, int B,
                                             long long N, void* cuda_stream)
{
    launch_count() = 0;
    if (!mip_shape_ok(TB, TH, TW, C, B, N)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0 || N == 0) return DIRT_OK;
    if (!texture || !indices || !derivatives || !out || (!pyramid && mip_levels(TH, TW) > 1)) return DIRT_ERR_NULL_POINTER;
    if (!aligned({texture, pyramid, indices, derivatives, out})) return DIRT_ERR_MISALIGNED;
    CUDA_TRY(launch_texture_trilinear_forward(texture, pyramid, indices, derivatives, out,
                                              make_tex_dims(TB, TH, TW, C, B, N, DIRT_TEXTURE_BILINEAR),
                                              (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" size_t dirt_texture_sample_trilinear_backward_bytes(int TB, int TH, int TW, int C, int B, long long N,
                                                               int deterministic)
{
    if (!mip_shape_ok(TB, TH, TW, C, B, N)) return 0;
    if (deterministic && (!texture_det_shape_ok(TB, TH, TW, C, B, N, DIRT_TEXTURE_BILINEAR) || (long long)B * N == 0)) return 0;
    const TexDims d = make_tex_dims(TB, TH, TW, C, B, N, DIRT_TEXTURE_BILINEAR);
    if (!deterministic && mip_levels(TH, TW) == 1) return 0;
    return carve_texture_mip_scratch(nullptr, d, deterministic != 0).bytes;
}

extern "C" int dirt_texture_sample_trilinear_backward(const float* texture, const float* pyramid, const float* indices,
                                                      const float* derivatives, const float* grad_out, float* grad_texture,
                                                      float* grad_indices, int TB, int TH, int TW, int C, int B, long long N,
                                                      int deterministic, void* scratch, size_t scratch_bytes,
                                                      void* cuda_stream)
{
    launch_count() = 0;
    if (!mip_shape_ok(TB, TH, TW, C, B, N)) return DIRT_ERR_BAD_SHAPE;
    if (deterministic && grad_texture && !texture_det_shape_ok(TB, TH, TW, C, B, N, DIRT_TEXTURE_BILINEAR))
        return DIRT_ERR_BAD_SHAPE;
    const TexDims d = make_tex_dims(TB, TH, TW, C, B, N, DIRT_TEXTURE_BILINEAR);
    const int L = mip_levels(TH, TW);
    if (d.total > 0) {
        if (!indices || !derivatives || !grad_out) return DIRT_ERR_NULL_POINTER;
        if (grad_indices && (!texture || (!pyramid && L > 1))) return DIRT_ERR_NULL_POINTER;
    }
    if (!aligned({texture, pyramid, indices, derivatives, grad_out, grad_texture, grad_indices})) return DIRT_ERR_MISALIGNED;
    // the scratch holds the pyramid's gradients (default) or the per-level passes (deterministic)
    const bool det = deterministic && grad_texture && d.total > 0;
    const bool uses_scratch = grad_texture && d.total > 0 && (det || L > 1);
    if (uses_scratch) {
        const int rc = scratch_check(scratch, scratch_bytes,
                                     dirt_texture_sample_trilinear_backward_bytes(TB, TH, TW, C, B, N, det));
        if (rc != DIRT_OK) return rc;
    }
    CUDA_TRY(launch_texture_trilinear_backward(texture, pyramid, indices, derivatives, grad_out, grad_texture, grad_indices, d,
                                               det, carve_texture_mip_scratch(uses_scratch ? scratch : nullptr, d, det),
                                               (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// ---- cube-map lookup ----

// S <= 2^14 keeps a padded face's texel index in int32; the atlas is six face blocks of the texture limits
static bool cubemap_shape_ok(int TB, int S, int C, int B, long long N, int mode)
{
    if (S <= 0 || S > (1 << 14)) return false;
    return texture_shape_ok(TB, S + 2, S + 2, C, B, N, mode) && (double)TB * 6 * (S + 2) * (S + 2) * C <= 4.0e18 &&
           (double)B * N * (C > 3 ? C : 3) <= 4.0e18;
}

static TexDims cubemap_dims(int TB, int S, int C, int B, long long N, int mode)
{
    return make_tex_dims(TB, S + 2, S + 2, C, B, N, mode);
}

extern "C" size_t dirt_cubemap_atlas_bytes(int TB, int S, int C)
{
    if (TB < 0 || !cubemap_shape_ok(TB, S, C, TB, 0, DIRT_TEXTURE_BILINEAR)) return 0;
    return sizeof(float) * 6 * (size_t)TB * (S + 2) * (S + 2) * C;
}

extern "C" int dirt_cubemap_sample(const float* cubemap, const float* directions, float* atlas, float* out, int TB, int S,
                                   int C, int B, long long N, int mode, void* cuda_stream)
{
    launch_count() = 0;
    if (!cubemap_shape_ok(TB, S, C, B, N, mode)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0 || N == 0) return DIRT_OK;
    const int rc = required_check({cubemap, directions, atlas, out});
    if (rc != DIRT_OK) return rc;
    CUDA_TRY(launch_cubemap_forward(cubemap, directions, atlas, out, cubemap_dims(TB, S, C, B, N, mode),
                                    (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" size_t dirt_cubemap_sample_backward_bytes(int TB, int S, int C, int B, long long N, int mode, int deterministic)
{
    if (!cubemap_shape_ok(TB, S, C, B, N, mode) || (long long)B * N == 0) return 0;
    if (deterministic && !texture_det_shape_ok(TB, S + 2, S + 2, C, B, N, mode)) return 0;
    return carve_cubemap_scratch(nullptr, cubemap_dims(TB, S, C, B, N, mode), deterministic != 0).bytes;
}

extern "C" int dirt_cubemap_sample_backward(const float* atlas, const float* directions, const float* grad_out,
                                            float* grad_cubemap, float* grad_directions, int TB, int S, int C, int B,
                                            long long N, int mode, int deterministic, void* scratch, size_t scratch_bytes,
                                            void* cuda_stream)
{
    launch_count() = 0;
    if (!cubemap_shape_ok(TB, S, C, B, N, mode)) return DIRT_ERR_BAD_SHAPE;
    if (deterministic && grad_cubemap && !texture_det_shape_ok(TB, S + 2, S + 2, C, B, N, mode)) return DIRT_ERR_BAD_SHAPE;
    const TexDims d = cubemap_dims(TB, S, C, B, N, mode);
    if (d.total > 0) {
        if (!directions || !grad_out) return DIRT_ERR_NULL_POINTER;
        if (grad_directions && mode == DIRT_TEXTURE_BILINEAR && !atlas) return DIRT_ERR_NULL_POINTER;
    }
    if (!aligned({atlas, directions, grad_out, grad_cubemap, grad_directions})) return DIRT_ERR_MISALIGNED;
    // the scratch holds the atlas's gradient (and the deterministic path's per-face passes)
    const bool det = deterministic && grad_cubemap && d.total > 0;
    const bool uses_scratch = grad_cubemap && d.total > 0;
    if (uses_scratch) {
        const int rc = scratch_check(scratch, scratch_bytes, dirt_cubemap_sample_backward_bytes(TB, S, C, B, N, mode, det));
        if (rc != DIRT_OK) return rc;
    }
    CUDA_TRY(launch_cubemap_backward(atlas, directions, grad_out, grad_cubemap, grad_directions, d, det,
                                     carve_cubemap_scratch(uses_scratch ? scratch : nullptr, d, det),
                                     (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// ---- mipmapped cube-map lookup ----

// the bilinear cube-map lookup's limits; the mip atlas is at most 4/3 of level 0's plus its borders
static bool cubemap_mip_shape_ok(int TB, int S, int C, int B, long long N)
{
    return cubemap_shape_ok(TB, S, C, B, N, DIRT_TEXTURE_BILINEAR) && (double)TB * 8 * (S + 2) * (S + 2) * C <= 4.0e18;
}

extern "C" size_t dirt_cubemap_mip_atlas_bytes(int TB, int S, int C)
{
    if (TB < 0 || !cubemap_mip_shape_ok(TB, S, C, TB, 0)) return 0;
    return sizeof(float) * cubemap_mip_atlas_texels(cubemap_dims(TB, S, C, TB, 0, DIRT_TEXTURE_BILINEAR)) * C;
}

extern "C" int dirt_cubemap_sample_trilinear(const float* cubemap, const float* directions, const float* lod, float* atlas,
                                             float* out, int TB, int S, int C, int B, long long N, void* cuda_stream)
{
    launch_count() = 0;
    if (!cubemap_mip_shape_ok(TB, S, C, B, N)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0 || N == 0) return DIRT_OK;
    const int rc = required_check({cubemap, directions, lod, atlas, out});
    if (rc != DIRT_OK) return rc;
    CUDA_TRY(launch_cubemap_mip_forward(cubemap, directions, lod, atlas, out,
                                        cubemap_dims(TB, S, C, B, N, DIRT_TEXTURE_BILINEAR), (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" size_t dirt_cubemap_sample_trilinear_backward_bytes(int TB, int S, int C, int B, long long N, int deterministic)
{
    if (!cubemap_mip_shape_ok(TB, S, C, B, N) || (long long)B * N == 0) return 0;
    if (deterministic && !texture_det_shape_ok(TB, S + 2, S + 2, C, B, N, DIRT_TEXTURE_BILINEAR)) return 0;
    return carve_cubemap_mip_scratch(nullptr, cubemap_dims(TB, S, C, B, N, DIRT_TEXTURE_BILINEAR), deterministic != 0).bytes;
}

extern "C" int dirt_cubemap_sample_trilinear_backward(const float* atlas, const float* directions, const float* lod,
                                                      const float* grad_out, float* grad_cubemap, float* grad_directions,
                                                      float* grad_lod, int TB, int S, int C, int B, long long N,
                                                      int deterministic, void* scratch, size_t scratch_bytes,
                                                      void* cuda_stream)
{
    launch_count() = 0;
    if (!cubemap_mip_shape_ok(TB, S, C, B, N)) return DIRT_ERR_BAD_SHAPE;
    if (deterministic && grad_cubemap && !texture_det_shape_ok(TB, S + 2, S + 2, C, B, N, DIRT_TEXTURE_BILINEAR))
        return DIRT_ERR_BAD_SHAPE;
    const TexDims d = cubemap_dims(TB, S, C, B, N, DIRT_TEXTURE_BILINEAR);
    if (d.total > 0) {
        if (!directions || !lod || !grad_out) return DIRT_ERR_NULL_POINTER;
        if ((grad_directions || grad_lod) && !atlas) return DIRT_ERR_NULL_POINTER;
    }
    if (!aligned({atlas, directions, lod, grad_out, grad_cubemap, grad_directions, grad_lod})) return DIRT_ERR_MISALIGNED;
    // the scratch holds the atlas's and the pyramid's gradients (and the deterministic path's per-level passes)
    const bool det = deterministic && grad_cubemap && d.total > 0;
    const bool uses_scratch = grad_cubemap && d.total > 0;
    if (uses_scratch) {
        const int rc = scratch_check(scratch, scratch_bytes, dirt_cubemap_sample_trilinear_backward_bytes(TB, S, C, B, N, det));
        if (rc != DIRT_OK) return rc;
    }
    CUDA_TRY(launch_cubemap_mip_backward(atlas, directions, lod, grad_out, grad_cubemap, grad_directions, grad_lod, d, det,
                                         carve_cubemap_mip_scratch(uses_scratch ? scratch : nullptr, d, det),
                                         (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// ---- split-sum GGX image-based lighting ----

// the mipmapped lookup's limits; the prefiltered levels, their normalisers and the texel table add less than the mip
// atlas again
static bool cubemap_ggx_shape_ok(int TB, int S, int C, int B, long long N)
{
    return cubemap_mip_shape_ok(TB, S, C, B, N) && (double)TB * 16 * (S + 2) * (S + 2) * (C + 4) <= 4.0e18;
}

extern "C" size_t dirt_cubemap_ggx_atlas_bytes(int TB, int S, int C)
{
    if (TB < 0 || !cubemap_ggx_shape_ok(TB, S, C, TB, 0)) return 0;
    return sizeof(float) * (size_t)ggx_layout(cubemap_dims(TB, S, C, TB, 0, DIRT_TEXTURE_BILINEAR)).floats;
}

extern "C" int dirt_cubemap_ggx_prefilter(const float* cubemap, float* atlas, int TB, int S, int C, void* cuda_stream)
{
    launch_count() = 0;
    if (TB < 0 || !cubemap_ggx_shape_ok(TB, S, C, TB, 0)) return DIRT_ERR_BAD_SHAPE;
    if (TB == 0) return DIRT_OK;
    const int rc = required_check({cubemap, atlas});
    if (rc != DIRT_OK) return rc;
    if ((uintptr_t)atlas % 16) return DIRT_ERR_MISALIGNED;
    CUDA_TRY(launch_ggx_prefilter(cubemap, atlas, cubemap_dims(TB, S, C, TB, 0, DIRT_TEXTURE_BILINEAR),
                                  (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_cubemap_sample_ggx(const float* cubemap, const float* directions, const float* lod, float* atlas,
                                       float* out, int TB, int S, int C, int B, long long N, void* cuda_stream)
{
    launch_count() = 0;
    if (!cubemap_ggx_shape_ok(TB, S, C, B, N)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0 || N == 0) return DIRT_OK;
    const int rc = required_check({cubemap, directions, lod, atlas, out});
    if (rc != DIRT_OK) return rc;
    if ((uintptr_t)atlas % 16) return DIRT_ERR_MISALIGNED;
    CUDA_TRY(launch_cubemap_ggx_forward(cubemap, directions, lod, atlas, out,
                                        cubemap_dims(TB, S, C, B, N, DIRT_TEXTURE_BILINEAR), (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" size_t dirt_cubemap_sample_ggx_backward_bytes(int TB, int S, int C, int B, long long N, int deterministic)
{
    if (!cubemap_ggx_shape_ok(TB, S, C, B, N) || (long long)B * N == 0) return 0;
    if (deterministic && !texture_det_shape_ok(TB, S + 2, S + 2, C, B, N, DIRT_TEXTURE_BILINEAR)) return 0;
    return carve_cubemap_ggx_scratch(nullptr, cubemap_dims(TB, S, C, B, N, DIRT_TEXTURE_BILINEAR), deterministic != 0).bytes;
}

extern "C" int dirt_cubemap_sample_ggx_backward(const float* atlas, const float* directions, const float* lod,
                                                const float* grad_out, float* grad_cubemap, float* grad_directions,
                                                float* grad_lod, int TB, int S, int C, int B, long long N, int deterministic,
                                                void* scratch, size_t scratch_bytes, void* cuda_stream)
{
    launch_count() = 0;
    if (!cubemap_ggx_shape_ok(TB, S, C, B, N)) return DIRT_ERR_BAD_SHAPE;
    if (deterministic && grad_cubemap && !texture_det_shape_ok(TB, S + 2, S + 2, C, B, N, DIRT_TEXTURE_BILINEAR))
        return DIRT_ERR_BAD_SHAPE;
    const TexDims d = cubemap_dims(TB, S, C, B, N, DIRT_TEXTURE_BILINEAR);
    if (d.total > 0) {
        if (!directions || !lod || !grad_out) return DIRT_ERR_NULL_POINTER;
        // the lookups read the atlas; the prefilter's adjoint reads its normalisers and texel table
        if ((grad_directions || grad_lod || grad_cubemap) && !atlas) return DIRT_ERR_NULL_POINTER;
    }
    if (!aligned({directions, lod, grad_out, grad_cubemap, grad_directions, grad_lod}) || (uintptr_t)atlas % 16)
        return DIRT_ERR_MISALIGNED;
    const bool det = deterministic && grad_cubemap && d.total > 0;
    const bool uses_scratch = grad_cubemap && d.total > 0;
    if (uses_scratch) {
        const int rc = scratch_check(scratch, scratch_bytes, dirt_cubemap_sample_ggx_backward_bytes(TB, S, C, B, N, det));
        if (rc != DIRT_OK) return rc;
    }
    CUDA_TRY(launch_cubemap_ggx_backward(atlas, directions, lod, grad_out, grad_cubemap, grad_directions, grad_lod, d, det,
                                         carve_cubemap_ggx_scratch(uses_scratch ? scratch : nullptr, d, det),
                                         (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// S <= 2^14 and the [TB, 6, S, S, C] elements within int64, as the cube-map lookup
static bool cubemap_sh_shape_ok(int TB, int S, int C)
{
    return TB >= 0 && S > 0 && S <= (1 << 14) && C > 0 && (double)TB * 6 * S * S * C <= 4.0e18;
}

extern "C" size_t dirt_cubemap_sh_project_bytes(int TB, int S, int C)
{
    return cubemap_sh_shape_ok(TB, S, C) && TB > 0 ? sh_project_scratch_bytes(TB, S, C) : 0;
}

extern "C" int dirt_cubemap_sh_project(const float* cubemap, float* coeffs, void* scratch, size_t scratch_bytes, int TB,
                                       int S, int C, void* cuda_stream)
{
    launch_count() = 0;
    if (!cubemap_sh_shape_ok(TB, S, C)) return DIRT_ERR_BAD_SHAPE;
    if (TB == 0) return DIRT_OK;
    if (!cubemap || !coeffs || !scratch) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)cubemap % 4 || (uintptr_t)coeffs % 4 || (uintptr_t)scratch % 256) return DIRT_ERR_MISALIGNED;
    if (scratch_bytes < sh_project_scratch_bytes(TB, S, C)) return DIRT_ERR_WORKSPACE_TOO_SMALL;
    CUDA_TRY(launch_sh_project(cubemap, coeffs, scratch, TB, S, C, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_cubemap_sh_project_backward(const float* grad_coeffs, float* grad_cubemap, void* scratch,
                                                size_t scratch_bytes, int TB, int S, int C, void* cuda_stream)
{
    launch_count() = 0;
    if (!cubemap_sh_shape_ok(TB, S, C)) return DIRT_ERR_BAD_SHAPE;
    if (TB == 0) return DIRT_OK;
    if (!grad_coeffs || !grad_cubemap || !scratch) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)grad_coeffs % 4 || (uintptr_t)grad_cubemap % 4 || (uintptr_t)scratch % 256) return DIRT_ERR_MISALIGNED;
    if (scratch_bytes < sh_project_scratch_bytes(TB, S, C)) return DIRT_ERR_WORKSPACE_TOO_SMALL;
    CUDA_TRY(launch_sh_project_backward(grad_coeffs, grad_cubemap, scratch, TB, S, C, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// ---- equirectangular panoramas to cube maps ----

// H, W <= 2^20 keep a sample's rows and columns within half a texel of its fp32 coordinates, and S * n at most
// 2^21 / pi + S < 2^20, so the sub-sample numerators 2k + 1 are exact in fp32; n <= 4096 keeps n^2 exact in fp32; the
// elements within int64
static bool latlong_shape_ok(int TB, int H, int W, int S, int C)
{
    if (TB < 0 || H < 1 || W < 1 || H > (1 << 20) || W > (1 << 20) || S < 1 || S > (1 << 14) || C < 1) return false;
    return latlong_samples(H, W, S) <= 4096 && (double)TB * H * W * C <= 4.0e18 && (double)TB * 6 * S * S * C <= 4.0e18;
}

extern "C" int dirt_latlong_samples(int H, int W, int S)
{
    if (H < 1 || W < 1 || S < 1) return 0;
    return latlong_samples(H, W, S);
}

extern "C" int dirt_latlong_to_cubemap(const float* panorama, float* cubemap, int TB, int H, int W, int S, int C,
                                       void* cuda_stream)
{
    launch_count() = 0;
    if (!latlong_shape_ok(TB, H, W, S, C)) return DIRT_ERR_BAD_SHAPE;
    if (TB == 0) return DIRT_OK;
    const int rc = required_check({panorama, cubemap});
    if (rc != DIRT_OK) return rc;
    CUDA_TRY(launch_latlong_forward(panorama, cubemap, TB, H, W, S, C, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_latlong_to_cubemap_backward(const float* grad_cubemap, float* grad_panorama, int TB, int H, int W,
                                                int S, int C, void* cuda_stream)
{
    launch_count() = 0;
    if (!latlong_shape_ok(TB, H, W, S, C)) return DIRT_ERR_BAD_SHAPE;
    if (TB == 0) return DIRT_OK;
    const int rc = required_check({grad_cubemap, grad_panorama});
    if (rc != DIRT_OK) return rc;
    CUDA_TRY(launch_latlong_backward(grad_cubemap, grad_panorama, TB, H, W, S, C, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_ggx_brdf_table(float* table, int N, void* cuda_stream)
{
    launch_count() = 0;
    if (N < 0 || N > 4096) return DIRT_ERR_BAD_SHAPE;
    if (N == 0) return DIRT_OK;
    const int rc = required_check({table});
    if (rc != DIRT_OK) return rc;
    CUDA_TRY(launch_ggx_brdf_table(table, N, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// ---- the fused per-point ops: reflectance, GGX, spherical harmonics and normal mapping ----------------------------

// element offsets of every per-point buffer stay below 2^62 (B * V rows of at most `width` floats plus the inputs' row
// strides), the chunk count within the grid's x limit
static bool points_shape_ok(int B, long long V, double width, std::initializer_list<long long> strides)
{
    if (B < 0 || V < 0) return false;
    for (long long s : strides) {
        if (s < 0) return false;
        width += s;
    }
    return (double)B * V * width <= 4.0e18 && light_chunks(V) <= 0x7fffffffll;
}

// the partial rows of the reflectance and GGX parameter gradients stay below 2^62 bytes
static bool light_partials_ok(int B, long long V, int C)
{
    return (double)B * light_chunks(V) * (LIGHT_FIXED_PARAMS + (double)C) * sizeof(float) <= 4.0e18;
}

// the partials workspace of the per-item parameter gradients, `need` bytes, set as *partial when it passes
static int partials_check(void* workspace, size_t workspace_bytes, size_t need, float** partial)
{
    const int rc = required_check({workspace});
    if (rc != DIRT_OK) return rc;
    if (workspace_bytes < need) return DIRT_ERR_WORKSPACE_TOO_SMALL;
    *partial = static_cast<float*>(workspace);
    return DIRT_OK;
}

static bool lighting_shape_ok(int model, int B, long long V, int C, long long sn, long long sp, long long sc)
{
    const bool known = model == DIRT_LIGHT_DIFFUSE_DIRECTIONAL || model == DIRT_LIGHT_SPECULAR_DIRECTIONAL ||
                       model == DIRT_LIGHT_DIFFUSE_POINT;
    return known && C > 0 && points_shape_ok(B, V, C > 3 ? C : 3, {sn, sp, sc}) && light_partials_ok(B, V, C);
}

extern "C" size_t dirt_lighting_workspace_bytes(int B, long long V, int C)
{
    if (B <= 0 || V <= 0 || C <= 0) return 0;
    return sizeof(float) * (size_t)B * (size_t)light_chunks(V) * (size_t)(LIGHT_FIXED_PARAMS + C);
}

static LightArgs make_light_args(int model, int double_sided, const float* normals, long long sn, const float* positions,
                                 long long sp, const float* colors, long long sc, const float* light, int light_per_item,
                                 const float* light_color, int light_color_per_item, const float* camera,
                                 int camera_per_item, const float* shininess, int shininess_per_item, int B, long long V,
                                 int C)
{
    LightArgs a = {};
    a.normals = normals; a.positions = positions; a.colors = colors;
    a.sn = sn; a.sp = sp; a.sc = sc;
    a.light = light; a.light_color = light_color; a.camera = camera; a.shininess = shininess;
    a.item_light = light_per_item != 0; a.item_color = light_color_per_item != 0;
    a.item_camera = camera_per_item != 0; a.item_shininess = shininess_per_item != 0;
    a.V = V; a.B = B; a.C = C; a.chunks = (int)light_chunks(V);
    a.model = model; a.double_sided = double_sided != 0;
    return a;
}

// the inputs a model reads are required, the others ignored
static int lighting_inputs_check(const LightArgs& a)
{
    if (a.model == DIRT_LIGHT_DIFFUSE_DIRECTIONAL) return required_check({a.normals, a.colors, a.light, a.light_color});
    if (a.model == DIRT_LIGHT_DIFFUSE_POINT)
        return required_check({a.normals, a.positions, a.colors, a.light, a.light_color});
    return required_check({a.normals, a.positions, a.colors, a.light, a.light_color, a.camera, a.shininess});
}

extern "C" int dirt_lighting_forward(int model, int double_sided, const float* normals, long long normals_stride,
                                     const float* positions, long long positions_stride, const float* colors,
                                     long long colors_stride, const float* light, int light_per_item,
                                     const float* light_color, int light_color_per_item, const float* camera,
                                     int camera_per_item, const float* shininess, int shininess_per_item, float* out,
                                     int B, long long V, int C, void* cuda_stream)
{
    launch_count() = 0;
    if (!lighting_shape_ok(model, B, V, C, normals_stride, positions_stride, colors_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    LightArgs a = make_light_args(model, double_sided, normals, normals_stride, positions, positions_stride, colors,
                                  colors_stride, light, light_per_item, light_color, light_color_per_item, camera,
                                  camera_per_item, shininess, shininess_per_item, B, V, C);
    a.out = out;
    int rc = lighting_inputs_check(a);
    if (rc == DIRT_OK) rc = required_check({out});
    if (rc != DIRT_OK) return rc;
    CUDA_TRY(launch_lighting_forward(a, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_lighting_backward(int model, int double_sided, const float* normals, long long normals_stride,
                                      const float* positions, long long positions_stride, const float* colors,
                                      long long colors_stride, const float* light, int light_per_item,
                                      const float* light_color, int light_color_per_item, const float* camera,
                                      int camera_per_item, const float* shininess, int shininess_per_item,
                                      const float* grad_out, float* grad_normals, float* grad_positions,
                                      float* grad_colors, float* grad_light, float* grad_light_color, float* grad_camera,
                                      float* grad_shininess, void* workspace, size_t workspace_bytes, int B, long long V,
                                      int C, void* cuda_stream)
{
    launch_count() = 0;
    if (!lighting_shape_ok(model, B, V, C, normals_stride, positions_stride, colors_stride)) return DIRT_ERR_BAD_SHAPE;
    LightArgs a = make_light_args(model, double_sided, normals, normals_stride, positions, positions_stride, colors,
                                  colors_stride, light, light_per_item, light_color, light_color_per_item, camera,
                                  camera_per_item, shininess, shininess_per_item, B, V, C);
    const bool sp = model == DIRT_LIGHT_SPECULAR_DIRECTIONAL;
    a.grad_out = grad_out;
    a.g_normals = grad_normals; a.g_colors = grad_colors; a.g_light = grad_light; a.g_light_color = grad_light_color;
    a.g_positions = model != DIRT_LIGHT_DIFFUSE_DIRECTIONAL ? grad_positions : nullptr;
    a.g_camera = sp ? grad_camera : nullptr;
    a.g_shininess = sp ? grad_shininess : nullptr;
    if (!aligned({a.g_normals, a.g_positions, a.g_colors, a.g_light, a.g_light_color, a.g_camera, a.g_shininess}))
        return DIRT_ERR_MISALIGNED;
    const bool params = a.g_light || a.g_light_color || a.g_camera || a.g_shininess;
    if ((long long)B * V > 0 && (params || a.g_normals || a.g_positions || a.g_colors)) {
        int rc = lighting_inputs_check(a);
        if (rc == DIRT_OK) rc = required_check({grad_out});
        if (rc == DIRT_OK && params)
            rc = partials_check(workspace, workspace_bytes, dirt_lighting_workspace_bytes(B, V, C), &a.partial);
        if (rc != DIRT_OK) return rc;
    }
    // with no points only the memsets of the wanted parameter gradients are enqueued
    CUDA_TRY(launch_lighting_backward(a, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

static bool ggx_shape_ok(int B, long long V, int C, long long sn, long long sp, long long sr, long long ss)
{
    return C > 0 && points_shape_ok(B, V, C > 3 ? C : 3, {sn, sp, sr, ss}) && light_partials_ok(B, V, C);
}

// LightArgs of a GGX call: the specular colour in place of the colours, model = point_light
static LightArgs make_ggx_args(int point_light, int double_sided, const float* normals, long long sn,
                               const float* positions, long long sp, const float* roughness, long long sr,
                               const float* specular, long long ss, const float* light, int light_per_item,
                               const float* light_color, int light_color_per_item, const float* camera,
                               int camera_per_item, int B, long long V, int C)
{
    LightArgs a = make_light_args(point_light != 0, double_sided, normals, sn, positions, sp, specular, ss, light,
                                  light_per_item, light_color, light_color_per_item, camera, camera_per_item, nullptr,
                                  0, B, V, C);
    a.roughness = roughness;
    a.sr = sr;
    return a;
}

extern "C" int dirt_ggx_lighting_forward(int point_light, int double_sided, const float* normals,
                                         long long normals_stride, const float* positions, long long positions_stride,
                                         const float* roughness, long long roughness_stride, const float* specular,
                                         long long specular_stride, const float* light, int light_per_item,
                                         const float* light_color, int light_color_per_item, const float* camera,
                                         int camera_per_item, float* out, int B, long long V, int C, void* cuda_stream)
{
    launch_count() = 0;
    if (!ggx_shape_ok(B, V, C, normals_stride, positions_stride, roughness_stride, specular_stride))
        return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    LightArgs a = make_ggx_args(point_light, double_sided, normals, normals_stride, positions, positions_stride,
                                roughness, roughness_stride, specular, specular_stride, light, light_per_item,
                                light_color, light_color_per_item, camera, camera_per_item, B, V, C);
    a.out = out;
    int rc = required_check({normals, positions, roughness, specular, light, light_color, camera});
    if (rc == DIRT_OK) rc = required_check({out});
    if (rc != DIRT_OK) return rc;
    CUDA_TRY(launch_ggx_forward(a, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_ggx_lighting_backward(int point_light, int double_sided, const float* normals,
                                          long long normals_stride, const float* positions, long long positions_stride,
                                          const float* roughness, long long roughness_stride, const float* specular,
                                          long long specular_stride, const float* light, int light_per_item,
                                          const float* light_color, int light_color_per_item, const float* camera,
                                          int camera_per_item, const float* grad_out, float* grad_normals,
                                          float* grad_positions, float* grad_roughness, float* grad_specular,
                                          float* grad_light, float* grad_light_color, float* grad_camera,
                                          void* workspace, size_t workspace_bytes, int B, long long V, int C,
                                          void* cuda_stream)
{
    launch_count() = 0;
    if (!ggx_shape_ok(B, V, C, normals_stride, positions_stride, roughness_stride, specular_stride))
        return DIRT_ERR_BAD_SHAPE;
    LightArgs a = make_ggx_args(point_light, double_sided, normals, normals_stride, positions, positions_stride,
                                roughness, roughness_stride, specular, specular_stride, light, light_per_item,
                                light_color, light_color_per_item, camera, camera_per_item, B, V, C);
    a.grad_out = grad_out;
    a.g_normals = grad_normals; a.g_positions = grad_positions; a.g_roughness = grad_roughness;
    a.g_colors = grad_specular; a.g_light = grad_light; a.g_light_color = grad_light_color; a.g_camera = grad_camera;
    if (!aligned({grad_normals, grad_positions, grad_roughness, grad_specular, grad_light, grad_light_color, grad_camera}))
        return DIRT_ERR_MISALIGNED;
    const bool params = grad_light || grad_light_color || grad_camera;
    if ((long long)B * V > 0 && (params || grad_normals || grad_positions || grad_roughness || grad_specular)) {
        int rc = required_check({normals, positions, roughness, specular, light, light_color, camera});
        if (rc == DIRT_OK) rc = required_check({grad_out});
        if (rc == DIRT_OK && params)
            rc = partials_check(workspace, workspace_bytes, dirt_lighting_workspace_bytes(B, V, C), &a.partial);
        if (rc != DIRT_OK) return rc;
    }
    // with no points only the memsets of the wanted parameter gradients are enqueued
    CUDA_TRY(launch_ggx_backward(a, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// 9*C an int, and the partial rows of the coefficient gradient below 2^62 bytes
static bool sh_shape_ok(int B, long long V, int C, long long sn, long long sa)
{
    return C > 0 && C <= (1 << 26) && points_shape_ok(B, V, C > 3 ? C : 3, {sn, sa}) &&
           (double)B * sh_chunks(V) * 9.0 * C * sizeof(float) <= 4.0e18;
}

extern "C" size_t dirt_sh_lighting_workspace_bytes(int B, long long V, int C)
{
    if (B <= 0 || V <= 0 || C <= 0) return 0;
    return sizeof(float) * (size_t)B * (size_t)sh_chunks(V) * (size_t)(9 * (size_t)C);
}

static ShArgs make_sh_args(const float* normals, long long sn, const float* albedo, long long sa, const float* coefficients,
                           int coefficients_per_item, int B, long long V, int C)
{
    ShArgs a = {};
    a.normals = normals; a.albedo = albedo; a.coefficients = coefficients;
    a.sn = sn; a.sa = sa;
    a.item_coef = coefficients_per_item != 0;
    a.V = V; a.B = B; a.C = C; a.chunks = (int)sh_chunks(V);
    return a;
}

extern "C" int dirt_sh_lighting_forward(const float* normals, long long normals_stride, const float* albedo,
                                        long long albedo_stride, const float* coefficients, int coefficients_per_item,
                                        float* out, int B, long long V, int C, void* cuda_stream)
{
    launch_count() = 0;
    if (!sh_shape_ok(B, V, C, normals_stride, albedo_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    ShArgs a = make_sh_args(normals, normals_stride, albedo, albedo_stride, coefficients, coefficients_per_item, B, V, C);
    a.out = out;
    int rc = required_check({normals, albedo, coefficients});
    if (rc == DIRT_OK) rc = required_check({out});
    if (rc != DIRT_OK) return rc;
    CUDA_TRY(launch_sh_lighting_forward(a, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_sh_lighting_backward(const float* normals, long long normals_stride, const float* albedo,
                                         long long albedo_stride, const float* coefficients, int coefficients_per_item,
                                         const float* grad_out, float* grad_normals, float* grad_albedo,
                                         float* grad_coefficients, void* workspace, size_t workspace_bytes, int B,
                                         long long V, int C, void* cuda_stream)
{
    launch_count() = 0;
    if (!sh_shape_ok(B, V, C, normals_stride, albedo_stride)) return DIRT_ERR_BAD_SHAPE;
    ShArgs a = make_sh_args(normals, normals_stride, albedo, albedo_stride, coefficients, coefficients_per_item, B, V, C);
    a.grad_out = grad_out;
    a.g_normals = grad_normals; a.g_albedo = grad_albedo; a.g_coef = grad_coefficients;
    if (!aligned({grad_normals, grad_albedo, grad_coefficients})) return DIRT_ERR_MISALIGNED;
    if ((long long)B * V > 0 && (grad_normals || grad_albedo || grad_coefficients)) {
        int rc = required_check({normals, albedo, coefficients});
        if (rc == DIRT_OK) rc = required_check({grad_out});
        if (rc == DIRT_OK && grad_coefficients)
            rc = partials_check(workspace, workspace_bytes, dirt_sh_lighting_workspace_bytes(B, V, C), &a.partial);
        if (rc != DIRT_OK) return rc;
    }
    // with no points only the memset of a wanted coefficient gradient is enqueued
    CUDA_TRY(launch_sh_lighting_backward(a, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// ---- shadow-map visibility (DESIGN.md §7.15) ------------------------------------------------------------------------

// the points as the other per-point ops', a map of at most 2^62 texel floats, the lookup's parameters in range, and the
// partial rows of the light-matrix gradient below 2^62 bytes
static bool shadow_shape_ok(int B, long long V, long long sp, int SH, int SW, int radius, float softness, float bias)
{
    return points_shape_ok(B, V, 3, {sp}) && SH > 0 && SW > 0 && (double)(B > 1 ? B : 1) * SH * SW * 2 <= 4.0e18 &&
           radius >= 0 && radius <= 3 && softness >= 0.f && bias >= 0.f && std::isfinite(softness) &&
           std::isfinite(bias) && (double)B * light_chunks(V) * SHADOW_MATRIX * sizeof(float) <= 4.0e18;
}

extern "C" size_t dirt_shadow_workspace_bytes(int B, long long V)
{
    if (B <= 0 || V <= 0) return 0;
    return sizeof(float) * (size_t)B * (size_t)light_chunks(V) * SHADOW_MATRIX;
}

static ShadowArgs make_shadow_args(const float* positions, long long sp, const float* light_matrix,
                                   const float* shadow_map, int per_item, int SH, int SW, int radius, float softness,
                                   float bias, int B, long long V)
{
    ShadowArgs a = {};
    a.positions = positions; a.sp = sp; a.matrix = light_matrix; a.map = shadow_map; a.per_item = per_item != 0;
    a.SH = SH; a.SW = SW; a.R = radius; a.softness = softness; a.bias = bias;
    a.V = V; a.B = B; a.chunks = (int)light_chunks(V);
    return a;
}

// the inputs, with the map's float2 texels 8-byte aligned
static int shadow_inputs_check(const ShadowArgs& a)
{
    const int rc = required_check({a.positions, a.matrix, a.map});
    if (rc != DIRT_OK) return rc;
    return (uintptr_t)a.map % 8 ? DIRT_ERR_MISALIGNED : DIRT_OK;
}

extern "C" int dirt_shadow_forward(const float* positions, long long positions_stride, const float* light_matrix,
                                   const float* shadow_map, int per_item, int SH, int SW, int radius, float softness,
                                   float bias, float* out, int B, long long V, void* cuda_stream)
{
    launch_count() = 0;
    if (!shadow_shape_ok(B, V, positions_stride, SH, SW, radius, softness, bias)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    ShadowArgs a = make_shadow_args(positions, positions_stride, light_matrix, shadow_map, per_item, SH, SW, radius,
                                    softness, bias, B, V);
    a.out = out;
    int rc = shadow_inputs_check(a);
    if (rc == DIRT_OK) rc = required_check({out});
    if (rc != DIRT_OK) return rc;
    CUDA_TRY(launch_shadow_forward(a, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// the deterministic backward's point ids and segment offsets are int32
static bool shadow_det_shape_ok(int B, long long V, int per_item, int SH, int SW)
{
    return (long long)B * V <= 0x7fffffffll && SH > 0 && SW > 0 &&
           shadow_det_keys(B, per_item != 0, SH, SW) + 2 <= 0x7fffffffll;
}

extern "C" size_t dirt_shadow_backward_deterministic_bytes(int B, long long V, int per_item, int SH, int SW)
{
    if (B <= 0 || V <= 0 || !shadow_det_shape_ok(B, V, per_item, SH, SW)) return 0;
    ShadowArgs a = {};
    a.B = B; a.V = V; a.per_item = per_item != 0; a.SH = SH; a.SW = SW;
    return carve_shadow_det_scratch(nullptr, a).bytes;
}

// Both shadow backward entries.  The deterministic one adds its int32 rule (shadow_det_shape_ok, a second
// DIRT_ERR_BAD_SHAPE check) and, when it sorts (a wanted map gradient and points), a scratch: NULL, then 4-byte
// alignment (not scratch_check's 256), then its size.
static int shadow_backward_impl(const float* positions, long long positions_stride, const float* light_matrix,
                                const float* shadow_map, int per_item, int SH, int SW, int radius, float softness,
                                float bias, const float* grad_out, float* grad_positions, float* grad_light_matrix,
                                float* grad_shadow_map, void* workspace, size_t workspace_bytes, bool deterministic,
                                void* scratch, size_t scratch_bytes, int B, long long V, void* cuda_stream)
{
    launch_count() = 0;
    if (!shadow_shape_ok(B, V, positions_stride, SH, SW, radius, softness, bias) ||
        (deterministic && !shadow_det_shape_ok(B, V, per_item, SH, SW)))
        return DIRT_ERR_BAD_SHAPE;
    ShadowArgs a = make_shadow_args(positions, positions_stride, light_matrix, shadow_map, per_item, SH, SW, radius,
                                    softness, bias, B, V);
    a.grad_out = grad_out;
    a.g_positions = grad_positions; a.g_matrix = grad_light_matrix; a.g_map = grad_shadow_map;
    if (!aligned({grad_positions, grad_light_matrix, grad_shadow_map}) || (uintptr_t)grad_shadow_map % 8)
        return DIRT_ERR_MISALIGNED;
    const bool sorts = deterministic && grad_shadow_map && (long long)B * V > 0;
    if ((long long)B * V > 0 && (grad_positions || grad_light_matrix || grad_shadow_map)) {
        int rc = shadow_inputs_check(a);
        if (rc == DIRT_OK) rc = required_check({grad_out});
        if (rc == DIRT_OK && grad_light_matrix)
            rc = partials_check(workspace, workspace_bytes, dirt_shadow_workspace_bytes(B, V), &a.partial);
        if (rc == DIRT_OK && sorts) {
            rc = required_check({scratch});
            if (rc == DIRT_OK && scratch_bytes < dirt_shadow_backward_deterministic_bytes(B, V, per_item, SH, SW))
                rc = DIRT_ERR_WORKSPACE_TOO_SMALL;
        }
        if (rc != DIRT_OK) return rc;
    }
    // with no points only the memsets of the wanted map and matrix gradients are enqueued
    if (deterministic)
        CUDA_TRY(launch_shadow_backward_deterministic(a, carve_shadow_det_scratch(sorts ? scratch : nullptr, a),
                                                      (cudaStream_t)cuda_stream));
    else
        CUDA_TRY(launch_shadow_backward(a, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_shadow_backward(const float* positions, long long positions_stride, const float* light_matrix,
                                    const float* shadow_map, int per_item, int SH, int SW, int radius, float softness,
                                    float bias, const float* grad_out, float* grad_positions, float* grad_light_matrix,
                                    float* grad_shadow_map, void* workspace, size_t workspace_bytes, int B, long long V,
                                    void* cuda_stream)
{
    return shadow_backward_impl(positions, positions_stride, light_matrix, shadow_map, per_item, SH, SW, radius,
                                softness, bias, grad_out, grad_positions, grad_light_matrix, grad_shadow_map, workspace,
                                workspace_bytes, false, nullptr, 0, B, V, cuda_stream);
}

extern "C" int dirt_shadow_backward_deterministic(const float* positions, long long positions_stride,
                                                  const float* light_matrix, const float* shadow_map, int per_item,
                                                  int SH, int SW, int radius, float softness, float bias,
                                                  const float* grad_out, float* grad_positions,
                                                  float* grad_light_matrix, float* grad_shadow_map, void* workspace,
                                                  size_t workspace_bytes, void* scratch, size_t scratch_bytes, int B,
                                                  long long V, void* cuda_stream)
{
    return shadow_backward_impl(positions, positions_stride, light_matrix, shadow_map, per_item, SH, SW, radius,
                                softness, bias, grad_out, grad_positions, grad_light_matrix, grad_shadow_map, workspace,
                                workspace_bytes, true, scratch, scratch_bytes, B, V, cuda_stream);
}

// element offsets of the vertex rows stay below 2^62; vertex ids and incidence ids (k*F + f) are int32
static bool normals_shape_ok(int mode, int B, long long V, long long F, long long stride)
{
    if (mode != DIRT_NORMALS_AVERAGE && mode != DIRT_NORMALS_PRE_SPLIT) return false;
    if (B < 0 || V < 0 || F < 0 || stride < 3) return false;
    if (V >= (1ll << 31) || 3 * F >= (1ll << 31)) return false;
    return (double)B * V * stride <= 4.0e18;
}

extern "C" size_t dirt_normals_workspace_bytes(int B, long long V, long long F)
{
    if (!normals_shape_ok(DIRT_NORMALS_AVERAGE, B, V, F, 3) || B == 0 || V == 0 || F == 0) return 0;
    return carve_normals_workspace(nullptr, B, V, F).bytes;
}

// The checks the eight mesh entries share, in order: the vertices, faces and workspace, NULL (the faces and workspace
// only when a workspace is needed: `need`, the entry's workspace size, is 0 exactly when F = 0 once B*V > 0) then
// 4-byte alignment (the workspace holds int32 adjacency and float gradients, read and written one element at a time, so
// not scratch_check's 256 bytes); the workspace's size; the other inputs and then `outs` (the output, or the incoming
// gradient and the gradients a backward requires), each by required_check.  Before it each entry makes its shape check
// and its early return, which differ:
// - the forwards and the normals and Laplacian backwards return DIRT_OK for B*V == 0 before they check anything else;
// - the tangents backward first checks the alignment of its gradients, which may be NULL, then returns DIRT_OK for
//   B*V == 0 or when no gradient is wanted;
// - the edge-term entries return DIRT_OK for B*F == 0, and handle V == 0 themselves (see below).
static int mesh_check(const float* vertices, const int32_t* faces, const void* workspace, size_t workspace_bytes,
                      size_t need, std::initializer_list<const void*> inputs, std::initializer_list<const void*> outs)
{
    if (!vertices || (need > 0 && (!faces || !workspace))) return DIRT_ERR_NULL_POINTER;
    if (!aligned({vertices, faces, workspace})) return DIRT_ERR_MISALIGNED;
    if (workspace_bytes < need) return DIRT_ERR_WORKSPACE_TOO_SMALL;
    const int rc = required_check(inputs);
    return rc != DIRT_OK ? rc : required_check(outs);
}

static NormalsArgs make_normals_args(int mode, const float* vertices, long long stride, const int32_t* faces, int B,
                                     long long V, long long F)
{
    NormalsArgs a = {};
    a.vertices = vertices; a.stride = stride; a.faces = faces;
    a.total = (long long)B * V; a.V = (int)V; a.F = (int)F; a.mode = mode;
    return a;
}

extern "C" int dirt_normals_forward(int mode, const float* vertices, long long vertex_stride, const int32_t* faces,
                                    float* normals, void* workspace, size_t workspace_bytes, int B, long long V, long long F,
                                    void* cuda_stream)
{
    launch_count() = 0;
    if (!normals_shape_ok(mode, B, V, F, vertex_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    const int rc = mesh_check(vertices, faces, workspace, workspace_bytes, dirt_normals_workspace_bytes(B, V, F), {},
                              {normals});
    if (rc != DIRT_OK) return rc;
    NormalsArgs a = make_normals_args(mode, vertices, vertex_stride, faces, B, V, F);
    a.out = normals;
    CUDA_TRY(launch_normals_forward(a, carve_normals_workspace(F > 0 ? workspace : nullptr, B, V, F),
                                    (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_normals_backward(int mode, const float* vertices, long long vertex_stride, const int32_t* faces,
                                     const float* grad_normals, float* grad_vertices, void* workspace,
                                     size_t workspace_bytes, int B, long long V, long long F, void* cuda_stream)
{
    launch_count() = 0;
    if (!normals_shape_ok(mode, B, V, F, vertex_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    const int rc = mesh_check(vertices, faces, workspace, workspace_bytes, dirt_normals_workspace_bytes(B, V, F), {},
                              {grad_normals, grad_vertices});
    if (rc != DIRT_OK) return rc;
    NormalsArgs a = make_normals_args(mode, vertices, vertex_stride, faces, B, V, F);
    a.grad = grad_normals;
    a.g_vertices = grad_vertices;
    CUDA_TRY(launch_normals_backward(a, carve_normals_workspace(F > 0 ? workspace : nullptr, B, V, F),
                                     (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// ---- the mesh Laplacian (DESIGN.md §7.16): the normals' arguments, checks and early returns ------------------------

static bool laplacian_shape_ok(int mode, int B, long long V, long long F, long long stride)
{
    return (mode == DIRT_LAPLACIAN_UNIFORM || mode == DIRT_LAPLACIAN_COTANGENT) &&
           normals_shape_ok(DIRT_NORMALS_AVERAGE, B, V, F, stride);
}

extern "C" size_t dirt_laplacian_workspace_bytes(int B, long long V, long long F)
{
    if (!normals_shape_ok(DIRT_NORMALS_AVERAGE, B, V, F, 3) || B == 0 || V == 0 || F == 0) return 0;
    return carve_normals_workspace(nullptr, B, V, F, 4).bytes;
}

extern "C" int dirt_laplacian_forward(int mode, const float* vertices, long long vertex_stride, const int32_t* faces,
                                      float* out, void* workspace, size_t workspace_bytes, int B, long long V, long long F,
                                      void* cuda_stream)
{
    launch_count() = 0;
    if (!laplacian_shape_ok(mode, B, V, F, vertex_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    const int rc = mesh_check(vertices, faces, workspace, workspace_bytes, dirt_laplacian_workspace_bytes(B, V, F), {},
                              {out});
    if (rc != DIRT_OK) return rc;
    NormalsArgs a = make_normals_args(mode, vertices, vertex_stride, faces, B, V, F);
    a.out = out;
    CUDA_TRY(launch_laplacian_forward(a, carve_normals_workspace(F > 0 ? workspace : nullptr, B, V, F, 4),
                                      (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_laplacian_backward(int mode, const float* vertices, long long vertex_stride, const int32_t* faces,
                                       const float* grad_out, float* grad_vertices, void* workspace,
                                       size_t workspace_bytes, int B, long long V, long long F, void* cuda_stream)
{
    launch_count() = 0;
    if (!laplacian_shape_ok(mode, B, V, F, vertex_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    const int rc = mesh_check(vertices, faces, workspace, workspace_bytes, dirt_laplacian_workspace_bytes(B, V, F), {},
                              {grad_out, grad_vertices});
    if (rc != DIRT_OK) return rc;
    NormalsArgs a = make_normals_args(mode, vertices, vertex_stride, faces, B, V, F);
    a.grad = grad_out;
    a.g_vertices = grad_vertices;
    CUDA_TRY(launch_laplacian_backward(a, carve_normals_workspace(F > 0 ? workspace : nullptr, B, V, F, 4),
                                       (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// ---- edge lengths and normal consistency (DESIGN.md §7.17): the Laplacian's arguments and checks ---------------------
// The output is per face, so the early returns differ: the forward launches nothing for B*F == 0, and V == 0 with
// F > 0 makes every face invalid, so it zeroes out.  The backward writes nothing for B*V == 0 and zeroes grad_vertices
// for F == 0.  All are decided before mesh_check, which requires a workspace whenever F > 0.

static bool edge_terms_shape_ok(int mode, int B, long long V, long long F, long long stride)
{
    return (mode == DIRT_EDGE_LENGTH || mode == DIRT_NORMAL_CONSISTENCY) &&
           normals_shape_ok(DIRT_NORMALS_AVERAGE, B, V, F, stride);
}

extern "C" size_t dirt_edge_terms_workspace_bytes(int B, long long V, long long F)
{
    if (!normals_shape_ok(DIRT_NORMALS_AVERAGE, B, V, F, 3) || B == 0 || V == 0 || F == 0) return 0;
    return carve_normals_workspace(nullptr, B, V, F, 3, true).bytes;
}

extern "C" int dirt_edge_terms_forward(int mode, const float* vertices, long long vertex_stride, const int32_t* faces,
                                       float* out, void* workspace, size_t workspace_bytes, int B, long long V,
                                       long long F, void* cuda_stream)
{
    launch_count() = 0;
    if (!edge_terms_shape_ok(mode, B, V, F, vertex_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * F == 0) return DIRT_OK;
    if (V == 0) {
        const int rc = required_check({out});
        if (rc != DIRT_OK) return rc;
        CUDA_TRY(cudaMemsetAsync(out, 0, sizeof(float) * 3 * (size_t)B * (size_t)F, (cudaStream_t)cuda_stream));
        return DIRT_OK;
    }
    const int rc = mesh_check(vertices, faces, workspace, workspace_bytes, dirt_edge_terms_workspace_bytes(B, V, F), {},
                              {out});
    if (rc != DIRT_OK) return rc;
    NormalsArgs a = make_normals_args(mode, vertices, vertex_stride, faces, B, V, F);
    a.out = out;
    CUDA_TRY(launch_edge_terms_forward(a, carve_normals_workspace(workspace, B, V, F, 3, true), (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_edge_terms_backward(int mode, const float* vertices, long long vertex_stride, const int32_t* faces,
                                        const float* grad_out, float* grad_vertices, void* workspace,
                                        size_t workspace_bytes, int B, long long V, long long F, void* cuda_stream)
{
    launch_count() = 0;
    if (!edge_terms_shape_ok(mode, B, V, F, vertex_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    if (F == 0) {   // no edges: no gradient reaches the vertices
        const int rc = required_check({grad_vertices});
        if (rc != DIRT_OK) return rc;
        CUDA_TRY(cudaMemsetAsync(grad_vertices, 0, sizeof(float) * 3 * (size_t)B * (size_t)V, (cudaStream_t)cuda_stream));
        return DIRT_OK;
    }
    const int rc = mesh_check(vertices, faces, workspace, workspace_bytes, dirt_edge_terms_workspace_bytes(B, V, F), {},
                              {grad_out, grad_vertices});
    if (rc != DIRT_OK) return rc;
    NormalsArgs a = make_normals_args(mode, vertices, vertex_stride, faces, B, V, F);
    a.grad = grad_out;
    a.g_vertices = grad_vertices;
    CUDA_TRY(launch_edge_terms_backward(a, carve_normals_workspace(workspace, B, V, F, 3, true), (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

// ---- vertex tangents and normal mapping (DESIGN.md §7.14) ----------------------------------------------------------

// as normals_shape_ok, with the uv and normal rows' strides and the uvs' item stride
static bool tangents_shape_ok(int B, long long V, long long F, long long vs, long long us, long long uis, long long ns)
{
    if (!normals_shape_ok(DIRT_NORMALS_AVERAGE, B, V, F, vs) || us < 2 || uis < 0 || ns < 3) return false;
    const double rows = (double)B * V;
    return rows * us + (double)B * uis <= 4.0e18 && rows * ns <= 4.0e18 && rows * 4 <= 4.0e18;
}

extern "C" size_t dirt_tangents_workspace_bytes(int B, long long V, long long F)
{
    return dirt_normals_workspace_bytes(B, V, F);
}

static TangentArgs make_tangent_args(const float* vertices, long long vertex_stride, const float* uvs, long long uv_stride,
                                     long long uv_item_stride, const float* normals, long long normals_stride,
                                     const int32_t* faces, int B, long long V, long long F)
{
    TangentArgs a = {};
    a.m = make_normals_args(DIRT_NORMALS_AVERAGE, vertices, vertex_stride, faces, B, V, F);
    a.uvs = uvs; a.uv_stride = uv_stride; a.uv_item_stride = uv_item_stride;
    a.normals = normals; a.normal_stride = normals_stride;
    return a;
}

extern "C" int dirt_tangents_forward(const float* vertices, long long vertex_stride, const float* uvs, long long uv_stride,
                                     long long uv_item_stride, const float* normals, long long normals_stride,
                                     const int32_t* faces, float* tangents, void* workspace, size_t workspace_bytes, int B,
                                     long long V, long long F, void* cuda_stream)
{
    launch_count() = 0;
    if (!tangents_shape_ok(B, V, F, vertex_stride, uv_stride, uv_item_stride, normals_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    const int rc = mesh_check(vertices, faces, workspace, workspace_bytes, dirt_tangents_workspace_bytes(B, V, F),
                              {uvs, normals}, {tangents});
    if (rc != DIRT_OK) return rc;
    TangentArgs a = make_tangent_args(vertices, vertex_stride, uvs, uv_stride, uv_item_stride, normals, normals_stride,
                                      faces, B, V, F);
    a.out = tangents;
    CUDA_TRY(launch_tangents_forward(a, carve_normals_workspace(F > 0 ? workspace : nullptr, B, V, F),
                                     (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_tangents_backward(const float* vertices, long long vertex_stride, const float* uvs, long long uv_stride,
                                      long long uv_item_stride, const float* normals, long long normals_stride,
                                      const int32_t* faces, const float* grad_tangents, float* grad_vertices,
                                      float* grad_uvs, float* grad_normals, void* workspace, size_t workspace_bytes, int B,
                                      long long V, long long F, void* cuda_stream)
{
    launch_count() = 0;
    if (!tangents_shape_ok(B, V, F, vertex_stride, uv_stride, uv_item_stride, normals_stride)) return DIRT_ERR_BAD_SHAPE;
    if (!aligned({grad_vertices, grad_uvs, grad_normals})) return DIRT_ERR_MISALIGNED;
    if ((long long)B * V == 0 || (!grad_vertices && !grad_uvs && !grad_normals)) return DIRT_OK;
    const int rc = mesh_check(vertices, faces, workspace, workspace_bytes, dirt_tangents_workspace_bytes(B, V, F),
                              {uvs, normals}, {grad_tangents});
    if (rc != DIRT_OK) return rc;
    TangentArgs a = make_tangent_args(vertices, vertex_stride, uvs, uv_stride, uv_item_stride, normals, normals_stride,
                                      faces, B, V, F);
    a.grad = grad_tangents;
    a.g_vertices = grad_vertices; a.g_uvs = grad_uvs; a.g_normals = grad_normals;
    CUDA_TRY(launch_tangents_backward(a, carve_normals_workspace(F > 0 ? workspace : nullptr, B, V, F),
                                      (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

static NormalMapArgs make_normal_map_args(const float* normals, long long sn, const float* tangents, long long st,
                                          const float* samples, long long sm, int B, long long V)
{
    NormalMapArgs a = {};
    a.normals = normals; a.tangents = tangents; a.samples = samples;
    a.sn = sn; a.st = st; a.sm = sm;
    a.B = B; a.V = V;
    return a;
}

extern "C" int dirt_normal_map_forward(const float* normals, long long normals_stride, const float* tangents,
                                       long long tangents_stride, const float* samples, long long samples_stride,
                                       float* out, int B, long long V, void* cuda_stream)
{
    launch_count() = 0;
    if (!points_shape_ok(B, V, 4, {normals_stride, tangents_stride, samples_stride})) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    NormalMapArgs a = make_normal_map_args(normals, normals_stride, tangents, tangents_stride, samples, samples_stride, B, V);
    int rc = required_check({normals, tangents, samples});
    if (rc == DIRT_OK) rc = required_check({out});
    if (rc != DIRT_OK) return rc;
    a.out = out;
    CUDA_TRY(launch_normal_map_forward(a, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_normal_map_backward(const float* normals, long long normals_stride, const float* tangents,
                                        long long tangents_stride, const float* samples, long long samples_stride,
                                        const float* grad_out, float* grad_normals, float* grad_tangents,
                                        float* grad_samples, int B, long long V, void* cuda_stream)
{
    launch_count() = 0;
    if (!points_shape_ok(B, V, 4, {normals_stride, tangents_stride, samples_stride})) return DIRT_ERR_BAD_SHAPE;
    if (!aligned({grad_normals, grad_tangents, grad_samples})) return DIRT_ERR_MISALIGNED;
    if ((long long)B * V == 0 || (!grad_normals && !grad_tangents && !grad_samples)) return DIRT_OK;
    NormalMapArgs a = make_normal_map_args(normals, normals_stride, tangents, tangents_stride, samples, samples_stride, B, V);
    int rc = required_check({normals, tangents, samples});
    if (rc == DIRT_OK) rc = required_check({grad_out});
    if (rc != DIRT_OK) return rc;
    a.grad_out = grad_out;
    a.g_normals = grad_normals; a.g_tangents = grad_tangents; a.g_samples = grad_samples;
    CUDA_TRY(launch_normal_map_backward(a, (cudaStream_t)cuda_stream));
    return DIRT_OK;
}

extern "C" int dirt_workspace_status(const void* workspace, size_t workspace_bytes, int B, int H, int W, int C, int V, int F,
                                     void* cuda_stream)
{
    if (!shape_ok(B, H, W, C, V, F)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0) return DIRT_OK;
    const int rc = scratch_check(workspace, workspace_bytes, dirt_workspace_bytes_min(B, H, W, C, V, F));
    if (rc != DIRT_OK) return rc;
    const RasterCall r = raster_call(workspace, B, H, W, C, V, F, cuda_stream);
    Header h;
    if (cudaMemcpyAsync(&h, r.ws.header, sizeof(h), cudaMemcpyDeviceToHost, r.stream) != cudaSuccess) return DIRT_ERR_CUDA;
    if (cudaStreamSynchronize(r.stream) != cudaSuccess) return DIRT_ERR_CUDA;
    return h.error ? DIRT_ERR_STALE_WORKSPACE : DIRT_OK;
}
