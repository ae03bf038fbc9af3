// api.cu -- the C ABI of libdirt_b200.so (include/dirt_b200.h): argument validation, workspace
// carving and kernel sequencing.  No device allocation, no host synchronisation, no global state
// other than a thread-local launch counter.
#include "../../include/dirt_b200.h"
#include "common.cuh"

using namespace dirt;

static_assert(BWD_SHARED_GEOMETRY == DIRT_BWD_SHARED_GEOMETRY && BWD_SKIP_POSITION == DIRT_BWD_SKIP_POSITION &&
              BWD_SKIP_COLOUR == DIRT_BWD_SKIP_COLOUR, "flag values of common.cuh and dirt_b200.h differ");

static thread_local int t_last_launches = 0;

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
}  // namespace dirt

extern "C" int dirt_kernel_timer_enable(int which)
{
    KernelTimer& t = kernel_timer();
    if (which < 0 || which > 2) return DIRT_ERR_BAD_SHAPE;
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

extern "C" int dirt_last_launch_count(void) { return t_last_launches; }

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

// needs_face_id_scratch: only a backward call without face ids derives them into the workspace's last block
static int check_workspace(void* workspace, size_t workspace_bytes, int B, int H, int W, int C, int V, int F,
                           bool needs_face_id_scratch = false)
{
    if (!workspace) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)workspace % 256 != 0) return DIRT_ERR_MISALIGNED;
    const size_t need = needs_face_id_scratch ? dirt_workspace_bytes(B, H, W, C, V, F) : dirt_workspace_bytes_min(B, H, W, C, V, F);
    if (workspace_bytes < need) return DIRT_ERR_WORKSPACE_TOO_SMALL;
    return DIRT_OK;
}

#define CUDA_TRY(expr)                                   \
    do {                                                 \
        cudaError_t e__ = (expr);                        \
        if (e__ != cudaSuccess) { t_last_launches = launches; return DIRT_ERR_CUDA; } \
    } while (0)

extern "C" int dirt_rasterise_forward(const float* background, const float* vertices, const float* vertex_colors,
                                      const int32_t* faces, float* pixels, int32_t* face_ids_out, int B, int H, int W,
                                      int C, int V, int F, void* workspace, size_t workspace_bytes, void* cuda_stream)
{
    int launches = 0;
    t_last_launches = 0;
    if (!shape_ok(B, H, W, C, V, F)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0) return DIRT_OK;
    if (!background || !pixels) return DIRT_ERR_NULL_POINTER;
    if ((V > 0 && (!vertices || !vertex_colors)) || (F > 0 && !faces)) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)vertices % 16 != 0) return DIRT_ERR_MISALIGNED;
    if ((uintptr_t)background % 4 || (uintptr_t)pixels % 4 || (uintptr_t)vertex_colors % 4 || (uintptr_t)faces % 4 ||
        (uintptr_t)face_ids_out % 4)
        return DIRT_ERR_MISALIGNED;
    int rc = check_workspace(workspace, workspace_bytes, B, H, W, C, V, F);
    if (rc != DIRT_OK) return rc;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const Workspace ws = carve_workspace(workspace, B, H, W, C, V, F);
    const Dims d = make_dims(B, H, W, C, V, F);
    CUDA_TRY(launch_setup_and_bin(vertices, faces, vertex_colors, ws, d, stream, &launches));
    CUDA_TRY(launch_raster_forward(vertices, background, vertex_colors, pixels, face_ids_out, ws, d, stream, &launches));
    t_last_launches = launches;
    return DIRT_OK;
}

extern "C" int dirt_rasterise_visibility(const float* vertices, const int32_t* faces, int32_t* face_ids, float* gbuffer,
                                         int B, int H, int W, int V, int F, void* workspace, size_t workspace_bytes,
                                         void* cuda_stream)
{
    int launches = 0;
    t_last_launches = 0;
    if (!shape_ok(B, H, W, 1, V, F)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0) return DIRT_OK;
    if ((V > 0 && !vertices) || (F > 0 && !faces)) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)vertices % 16 != 0 || (uintptr_t)gbuffer % 16 != 0 || (uintptr_t)face_ids % 4 != 0)
        return DIRT_ERR_MISALIGNED;
    int rc = check_workspace(workspace, workspace_bytes, B, H, W, 1, V, F);
    if (rc != DIRT_OK) return rc;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const Workspace ws = carve_workspace(workspace, B, H, W, 1, V, F);
    const Dims d = make_dims(B, H, W, 1, V, F);
    CUDA_TRY(launch_setup_and_bin(vertices, faces, nullptr, ws, d, stream, &launches));
    CUDA_TRY(launch_raster_visibility(vertices, face_ids, gbuffer, ws, d, stream, &launches));
    t_last_launches = launches;
    return DIRT_OK;
}

static int backward_impl(const float* vertices, const int32_t* faces, const float* pixels, const float* grad_pixels,
                         const int32_t* face_ids, float* grad_background, float* grad_vertices, float* grad_vertex_colors,
                         int B, int H, int W, int C, int V, int F, const int* channel_groups, int n_groups,
                         int workspace_holds_setup, int flags, void* workspace, size_t workspace_bytes, void* cuda_stream,
                         bool deterministic = false, void* scratch = nullptr, size_t scratch_bytes = 0)
{
    int launches = 0;
    t_last_launches = 0;
    if (!shape_ok(B, H, W, C, V, F)) return DIRT_ERR_BAD_SHAPE;
    if (V > (1 << 24)) return DIRT_ERR_TOO_MANY_VERTICES;
    if (flags & ~(DIRT_BWD_SHARED_GEOMETRY | DIRT_BWD_SKIP_POSITION | DIRT_BWD_SKIP_COLOUR)) return DIRT_ERR_BAD_SHAPE;
    GroupSpec groups;
    int rc = make_groups(C, channel_groups, n_groups, &groups);
    if (rc != DIRT_OK) return rc;
    if (B == 0) return DIRT_OK;
    if (!grad_pixels) return DIRT_ERR_NULL_POINTER;
    if (!(flags & DIRT_BWD_SKIP_POSITION) && !pixels) return DIRT_ERR_NULL_POINTER;
    if (!(flags & DIRT_BWD_SKIP_COLOUR) && !grad_background) return DIRT_ERR_NULL_POINTER;
    if ((V > 0 && (!vertices || !grad_vertices || !grad_vertex_colors)) || (F > 0 && !faces)) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)vertices % 16 != 0 || (uintptr_t)grad_vertices % 16 != 0) return DIRT_ERR_MISALIGNED;
    if ((uintptr_t)pixels % 4 || (uintptr_t)grad_pixels % 4 || (uintptr_t)grad_background % 4 ||
        (uintptr_t)grad_vertex_colors % 4 || (uintptr_t)faces % 4 || (uintptr_t)face_ids % 4)
        return DIRT_ERR_MISALIGNED;
    rc = check_workspace(workspace, workspace_bytes, B, H, W, C, V, F, face_ids == nullptr);
    if (rc != DIRT_OK) return rc;
    if (deterministic) {
        if (!scratch) return DIRT_ERR_NULL_POINTER;
        if ((uintptr_t)scratch % 256 != 0) return DIRT_ERR_MISALIGNED;
        if (scratch_bytes < dirt_rasterise_backward_deterministic_bytes(B, H, W, C, V, F)) return DIRT_ERR_WORKSPACE_TOO_SMALL;
    }
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    const Workspace ws = carve_workspace(workspace, B, H, W, C, V, F);
    const Dims d = make_dims(B, H, W, C, V, F);
    const int32_t* ids = face_ids;
    // the tile coverage flags in the workspace describe `ids` when the raster kernel that produced them ran on this workspace
    const bool flags_valid = !ids || workspace_holds_setup;
    unsigned long long expect_tag = 0;
    if (!ids) {
        // no cached visibility: re-derive it exactly as the forward pass does
        CUDA_TRY(launch_setup_and_bin(vertices, faces, nullptr, ws, d, stream, &launches));
        CUDA_TRY(launch_raster_visibility(vertices, ws.face_ids, nullptr, ws, d, stream, &launches));
        ids = ws.face_ids;
    } else if (!workspace_holds_setup) {
        CUDA_TRY(launch_setup_only(vertices, faces, ws, d, stream, &launches));
    } else {
        // a promise: checked on the device against the tag the setup pass left in the workspace
        expect_tag = workspace_tag(vertices, faces, B, H, W, V, F);
    }
    if (deterministic)
        CUDA_TRY(launch_backward_deterministic(vertices, faces, pixels, grad_pixels, ids, grad_background, grad_vertices,
                                               grad_vertex_colors, ws, d, groups, flags, expect_tag,
                                               carve_det_scratch(scratch, B, H, W, C, V, F), stream, &launches));
    else
        CUDA_TRY(launch_backward(vertices, pixels, grad_pixels, ids, grad_background, grad_vertices, grad_vertex_colors, ws, d,
                                 groups, flags_valid, flags, expect_tag, stream, &launches));
    t_last_launches = launches;
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

// the adjacency's corner ids b*3F + k*F + f are int32
static bool deterministic_shape_ok(int B, int H, int W, int C, int V, int F)
{
    return shape_ok(B, H, W, C, V, F) && 3ll * B * F <= (1ll << 31) - 1;
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
    t_last_launches = 0;
    if (!deterministic_shape_ok(B, H, W, C, V, F)) return DIRT_ERR_BAD_SHAPE;
    return backward_impl(vertices, faces, pixels, grad_pixels, face_ids, grad_background, grad_vertices, grad_vertex_colors, B, H,
                         W, C, V, F, channel_groups, n_groups, workspace_holds_setup, flags, workspace, workspace_bytes,
                         cuda_stream, true, scratch, scratch_bytes);
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
    int launches = 0;
    t_last_launches = 0;
    if (!texture_shape_ok(TB, TH, TW, C, B, N, mode)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0 || N == 0) return DIRT_OK;
    if (!texture || !indices || !out) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)texture % 4 || (uintptr_t)indices % 4 || (uintptr_t)out % 4) return DIRT_ERR_MISALIGNED;
    CUDA_TRY(launch_texture_forward(texture, indices, out, make_tex_dims(TB, TH, TW, C, B, N, mode), (cudaStream_t)cuda_stream,
                                    &launches));
    t_last_launches = launches;
    return DIRT_OK;
}

extern "C" int dirt_texture_sample_backward(const float* texture, const float* indices, const float* grad_out,
                                            float* grad_texture, float* grad_indices, int TB, int TH, int TW, int C, int B,
                                            long long N, int mode, void* cuda_stream)
{
    int launches = 0;
    t_last_launches = 0;
    if (!texture_shape_ok(TB, TH, TW, C, B, N, mode)) return DIRT_ERR_BAD_SHAPE;
    const TexDims d = make_tex_dims(TB, TH, TW, C, B, N, mode);
    if (d.total > 0) {
        if (!indices || !grad_out) return DIRT_ERR_NULL_POINTER;
        if (grad_indices && mode == DIRT_TEXTURE_BILINEAR && !texture) return DIRT_ERR_NULL_POINTER;
    }
    if ((uintptr_t)texture % 4 || (uintptr_t)indices % 4 || (uintptr_t)grad_out % 4 || (uintptr_t)grad_texture % 4 ||
        (uintptr_t)grad_indices % 4)
        return DIRT_ERR_MISALIGNED;
    // with no lookups only the memset of grad_texture is enqueued
    CUDA_TRY(launch_texture_backward(texture, indices, grad_out, grad_texture, grad_indices, d, (cudaStream_t)cuda_stream,
                                     &launches));
    t_last_launches = launches;
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
    int launches = 0;
    t_last_launches = 0;
    if (!texture_det_shape_ok(TB, TH, TW, C, B, N, mode)) return DIRT_ERR_BAD_SHAPE;
    const TexDims d = make_tex_dims(TB, TH, TW, C, B, N, mode);
    if (d.total > 0) {
        if (!indices || !grad_out) return DIRT_ERR_NULL_POINTER;
        if (grad_indices && mode == DIRT_TEXTURE_BILINEAR && !texture) return DIRT_ERR_NULL_POINTER;
    }
    if ((uintptr_t)texture % 4 || (uintptr_t)indices % 4 || (uintptr_t)grad_out % 4 || (uintptr_t)grad_texture % 4 ||
        (uintptr_t)grad_indices % 4)
        return DIRT_ERR_MISALIGNED;
    // only the texture gradient of a call with lookups sorts them
    const bool sorts = grad_texture && d.total > 0;
    if (sorts) {
        if (!scratch) return DIRT_ERR_NULL_POINTER;
        if ((uintptr_t)scratch % 256) return DIRT_ERR_MISALIGNED;
        if (scratch_bytes < dirt_texture_sample_backward_deterministic_bytes(TB, TH, TW, C, B, N, mode))
            return DIRT_ERR_WORKSPACE_TOO_SMALL;
    }
    CUDA_TRY(launch_texture_backward_deterministic(texture, indices, grad_out, grad_texture, grad_indices, d,
                                                   carve_texture_det_scratch(sorts ? scratch : nullptr, d),
                                                   (cudaStream_t)cuda_stream, &launches));
    t_last_launches = launches;
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
    int launches = 0;
    t_last_launches = 0;
    if (TB < 0 || !texture_shape_ok(TB, TH, TW, C, TB, 0, DIRT_TEXTURE_BILINEAR)) return DIRT_ERR_BAD_SHAPE;
    if (TB == 0 || mip_levels(TH, TW) == 1) return DIRT_OK;
    if (!texture || !pyramid) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)texture % 4 || (uintptr_t)pyramid % 4) return DIRT_ERR_MISALIGNED;
    CUDA_TRY(launch_texture_mip_build(texture, pyramid, make_tex_dims(TB, TH, TW, C, TB, 0, DIRT_TEXTURE_BILINEAR),
                                      (cudaStream_t)cuda_stream, &launches));
    t_last_launches = launches;
    return DIRT_OK;
}

extern "C" int dirt_texture_sample_trilinear(const float* texture, const float* pyramid, const float* indices,
                                             const float* derivatives, float* out, int TB, int TH, int TW, int C, int B,
                                             long long N, void* cuda_stream)
{
    int launches = 0;
    t_last_launches = 0;
    if (!mip_shape_ok(TB, TH, TW, C, B, N)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0 || N == 0) return DIRT_OK;
    if (!texture || !indices || !derivatives || !out || (!pyramid && mip_levels(TH, TW) > 1)) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)texture % 4 || (uintptr_t)pyramid % 4 || (uintptr_t)indices % 4 || (uintptr_t)derivatives % 4 ||
        (uintptr_t)out % 4)
        return DIRT_ERR_MISALIGNED;
    CUDA_TRY(launch_texture_trilinear_forward(texture, pyramid, indices, derivatives, out,
                                              make_tex_dims(TB, TH, TW, C, B, N, DIRT_TEXTURE_BILINEAR),
                                              (cudaStream_t)cuda_stream, &launches));
    t_last_launches = launches;
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
    int launches = 0;
    t_last_launches = 0;
    if (!mip_shape_ok(TB, TH, TW, C, B, N)) return DIRT_ERR_BAD_SHAPE;
    if (deterministic && grad_texture && !texture_det_shape_ok(TB, TH, TW, C, B, N, DIRT_TEXTURE_BILINEAR))
        return DIRT_ERR_BAD_SHAPE;
    const TexDims d = make_tex_dims(TB, TH, TW, C, B, N, DIRT_TEXTURE_BILINEAR);
    const int L = mip_levels(TH, TW);
    if (d.total > 0) {
        if (!indices || !derivatives || !grad_out) return DIRT_ERR_NULL_POINTER;
        if (grad_indices && (!texture || (!pyramid && L > 1))) return DIRT_ERR_NULL_POINTER;
    }
    if ((uintptr_t)texture % 4 || (uintptr_t)pyramid % 4 || (uintptr_t)indices % 4 || (uintptr_t)derivatives % 4 ||
        (uintptr_t)grad_out % 4 || (uintptr_t)grad_texture % 4 || (uintptr_t)grad_indices % 4)
        return DIRT_ERR_MISALIGNED;
    // the scratch holds the pyramid's gradients (default) or the per-level passes (deterministic)
    const bool det = deterministic && grad_texture && d.total > 0;
    const bool uses_scratch = grad_texture && d.total > 0 && (det || L > 1);
    if (uses_scratch) {
        if (!scratch) return DIRT_ERR_NULL_POINTER;
        if ((uintptr_t)scratch % 256) return DIRT_ERR_MISALIGNED;
        if (scratch_bytes < dirt_texture_sample_trilinear_backward_bytes(TB, TH, TW, C, B, N, det)) return DIRT_ERR_WORKSPACE_TOO_SMALL;
    }
    CUDA_TRY(launch_texture_trilinear_backward(texture, pyramid, indices, derivatives, grad_out, grad_texture, grad_indices, d,
                                               det, carve_texture_mip_scratch(uses_scratch ? scratch : nullptr, d, det),
                                               (cudaStream_t)cuda_stream, &launches));
    t_last_launches = launches;
    return DIRT_OK;
}

// element offsets of every per-point buffer stay below 2^62, the chunk count within the grid's x limit
static bool lighting_shape_ok(int model, int B, long long V, int C, long long sn, long long sp, long long sc)
{
    if (model != DIRT_LIGHT_DIFFUSE_DIRECTIONAL && model != DIRT_LIGHT_SPECULAR_DIRECTIONAL &&
        model != DIRT_LIGHT_DIFFUSE_POINT)
        return false;
    if (B < 0 || V < 0 || C <= 0 || sn < 0 || sp < 0 || sc < 0) return false;
    const double limit = 4.0e18, rows = (double)B * V;
    const double widest = (double)(C > 3 ? C : 3) + sn + sp + sc;
    if (rows * widest > limit || light_chunks(V) > 0x7fffffffll) return false;
    if ((double)B * light_chunks(V) * (LIGHT_FIXED_PARAMS + (double)C) * sizeof(float) > limit) return false;
    return true;
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
    const bool pos = a.model != DIRT_LIGHT_DIFFUSE_DIRECTIONAL, sp = a.model == DIRT_LIGHT_SPECULAR_DIRECTIONAL;
    if (!a.normals || !a.colors || !a.light || !a.light_color || (pos && !a.positions) || (sp && (!a.camera || !a.shininess)))
        return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)a.normals % 4 || (uintptr_t)a.colors % 4 || (uintptr_t)a.light % 4 || (uintptr_t)a.light_color % 4 ||
        (pos && (uintptr_t)a.positions % 4) || (sp && ((uintptr_t)a.camera % 4 || (uintptr_t)a.shininess % 4)))
        return DIRT_ERR_MISALIGNED;
    return DIRT_OK;
}

extern "C" int dirt_lighting_forward(int model, int double_sided, const float* normals, long long normals_stride,
                                     const float* positions, long long positions_stride, const float* colors,
                                     long long colors_stride, const float* light, int light_per_item,
                                     const float* light_color, int light_color_per_item, const float* camera,
                                     int camera_per_item, const float* shininess, int shininess_per_item, float* out,
                                     int B, long long V, int C, void* cuda_stream)
{
    int launches = 0;
    t_last_launches = 0;
    if (!lighting_shape_ok(model, B, V, C, normals_stride, positions_stride, colors_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    LightArgs a = make_light_args(model, double_sided, normals, normals_stride, positions, positions_stride, colors,
                                  colors_stride, light, light_per_item, light_color, light_color_per_item, camera,
                                  camera_per_item, shininess, shininess_per_item, B, V, C);
    a.out = out;
    const int rc = lighting_inputs_check(a);
    if (rc != DIRT_OK) return rc;
    if (!out) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)out % 4) return DIRT_ERR_MISALIGNED;
    CUDA_TRY(launch_lighting_forward(a, (cudaStream_t)cuda_stream, &launches));
    t_last_launches = launches;
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
    int launches = 0;
    t_last_launches = 0;
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
    float* outs[] = {a.g_normals, a.g_positions, a.g_colors, a.g_light, a.g_light_color, a.g_camera, a.g_shininess};
    for (float* p : outs)
        if ((uintptr_t)p % 4) return DIRT_ERR_MISALIGNED;
    const bool params = a.g_light || a.g_light_color || a.g_camera || a.g_shininess;
    if ((long long)B * V > 0 && (params || a.g_normals || a.g_positions || a.g_colors)) {
        int rc = lighting_inputs_check(a);
        if (rc != DIRT_OK) return rc;
        if (!grad_out) return DIRT_ERR_NULL_POINTER;
        if ((uintptr_t)grad_out % 4) return DIRT_ERR_MISALIGNED;
        if (params) {
            if (!workspace) return DIRT_ERR_NULL_POINTER;
            if ((uintptr_t)workspace % 4) return DIRT_ERR_MISALIGNED;
            if (workspace_bytes < dirt_lighting_workspace_bytes(B, V, C)) return DIRT_ERR_WORKSPACE_TOO_SMALL;
            a.partial = static_cast<float*>(workspace);
        }
    }
    // with no points only the memsets of the wanted parameter gradients are enqueued
    CUDA_TRY(launch_lighting_backward(a, (cudaStream_t)cuda_stream, &launches));
    t_last_launches = launches;
    return DIRT_OK;
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

static int normals_check(const float* vertices, const int32_t* faces, const void* workspace, size_t workspace_bytes,
                         int B, long long V, long long F)
{
    if (!vertices || (F > 0 && (!faces || !workspace))) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)vertices % 4 || (uintptr_t)faces % 4 || (uintptr_t)workspace % 4) return DIRT_ERR_MISALIGNED;
    if (workspace_bytes < dirt_normals_workspace_bytes(B, V, F)) return DIRT_ERR_WORKSPACE_TOO_SMALL;
    return DIRT_OK;
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
    int launches = 0;
    t_last_launches = 0;
    if (!normals_shape_ok(mode, B, V, F, vertex_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    const int rc = normals_check(vertices, faces, workspace, workspace_bytes, B, V, F);
    if (rc != DIRT_OK) return rc;
    if (!normals) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)normals % 4) return DIRT_ERR_MISALIGNED;
    NormalsArgs a = make_normals_args(mode, vertices, vertex_stride, faces, B, V, F);
    a.out = normals;
    CUDA_TRY(launch_normals_forward(a, carve_normals_workspace(F > 0 ? workspace : nullptr, B, V, F),
                                    (cudaStream_t)cuda_stream, &launches));
    t_last_launches = launches;
    return DIRT_OK;
}

extern "C" int dirt_normals_backward(int mode, const float* vertices, long long vertex_stride, const int32_t* faces,
                                     const float* grad_normals, float* grad_vertices, void* workspace,
                                     size_t workspace_bytes, int B, long long V, long long F, void* cuda_stream)
{
    int launches = 0;
    t_last_launches = 0;
    if (!normals_shape_ok(mode, B, V, F, vertex_stride)) return DIRT_ERR_BAD_SHAPE;
    if ((long long)B * V == 0) return DIRT_OK;
    const int rc = normals_check(vertices, faces, workspace, workspace_bytes, B, V, F);
    if (rc != DIRT_OK) return rc;
    if (!grad_normals || !grad_vertices) return DIRT_ERR_NULL_POINTER;
    if ((uintptr_t)grad_normals % 4 || (uintptr_t)grad_vertices % 4) return DIRT_ERR_MISALIGNED;
    NormalsArgs a = make_normals_args(mode, vertices, vertex_stride, faces, B, V, F);
    a.grad = grad_normals;
    a.g_vertices = grad_vertices;
    CUDA_TRY(launch_normals_backward(a, carve_normals_workspace(F > 0 ? workspace : nullptr, B, V, F),
                                     (cudaStream_t)cuda_stream, &launches));
    t_last_launches = launches;
    return DIRT_OK;
}

extern "C" int dirt_workspace_status(const void* workspace, size_t workspace_bytes, int B, int H, int W, int C, int V, int F,
                                     void* cuda_stream)
{
    if (!shape_ok(B, H, W, C, V, F)) return DIRT_ERR_BAD_SHAPE;
    if (B == 0) return DIRT_OK;
    int rc = check_workspace(const_cast<void*>(workspace), workspace_bytes, B, H, W, C, V, F);
    if (rc != DIRT_OK) return rc;
    const Workspace ws = carve_workspace(const_cast<void*>(workspace), B, H, W, C, V, F);
    Header h;
    cudaStream_t stream = (cudaStream_t)cuda_stream;
    if (cudaMemcpyAsync(&h, ws.header, sizeof(h), cudaMemcpyDeviceToHost, stream) != cudaSuccess) return DIRT_ERR_CUDA;
    if (cudaStreamSynchronize(stream) != cudaSuccess) return DIRT_ERR_CUDA;
    return h.error ? DIRT_ERR_STALE_WORKSPACE : DIRT_OK;
}
