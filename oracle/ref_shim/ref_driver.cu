// ref_driver.cu -- runs the reference's OWN gradient kernel on a caller-supplied G-buffer.
//
// TEST INFRASTRUCTURE (oracle/_ref).  The Makefile compiles the reference's csrc/rasterise_grad_egl.cu UNMODIFIED
// (against the stand-in headers in this directory) together with this file into oracle/_ref/libdirt_ref_grad.so.
// This file only does what RasteriseGradOpGpu::Compute does around launch_grad_assembly
// (csrc/rasterise_grad_egl.cpp:381-472): allocate the four outputs, lay the per-pixel (barycentrics, clip_w) and
// vertex-index images out as the tiled, y-up RGBA32F framebuffer textures GL would have rendered
// (frame placement :405-411,436-437; clear values :442-445; indices stored as floats, csrc/shaders.cpp:71), wrap
// them in CUDA arrays and call the reference's launch_grad_assembly.  All arithmetic that produces a gradient is
// the reference's.
//
// The G-buffer is an INPUT: in the reference it comes from the OpenGL driver, here from whichever
// visibility implementation is being pinned (the CPU oracle's, in tests/ and tests/golden/make_ref_golden.py).
#include "tensorflow/core/framework/tensor.h"
#include "tensorflow/core/util/cuda_launch_config.h"

#include "rasterise_grad_common.h"   // the reference's header (csrc/), found through -I $(REFERENCE)/csrc

#include <algorithm>
#include <cstdint>
#include <vector>

namespace {

struct DeviceBuffer {
    void* p = nullptr;
    cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 4); }
    ~DeviceBuffer() { if (p) cudaFree(p); }
};

struct DeviceArray {
    cudaArray_t a = nullptr;
    ~DeviceArray() { if (a) cudaFreeArray(a); }
};

}  // namespace

#define TRY(expr)                                        \
    do {                                                 \
        cudaError_t e__ = (expr);                        \
        if (e__ != cudaSuccess) {                        \
            std::fprintf(stderr, "ref_driver: %s failed: %s\n", #expr, cudaGetErrorString(e__)); \
            return -(int)e__;                            \
        }                                                \
    } while (0)

// All pointers are HOST pointers.  Layouts are the op's (row-major, channels last, row 0 = top of the image):
//   gbuffer [B,H,W,4] = (bary0, bary1, bary2, clip_w), (-1,-1,-1,+inf) where uncovered
//   vertex_ids [B,H,W,3] = the visible face's three vertex indices, -1 where uncovered
//   pixels, grad_pixels, grad_background [B,H,W,C] with C = 1 or 3 (one native-op call, csrc/hwc.h:27)
//   vertices, grad_vertices [B,V,4]; grad_vertex_colors [B,V,C]; debug_thingy [B,H,W,3] (may be NULL)
// Returns 0 on success, DIRT_REF_BAD_ARGS for invalid sizes, DIRT_REF_FRAME_TOO_LARGE when the tiled framebuffer is
// larger than a 2D surface can be on this device (nothing is allocated then), a negated cudaError_t otherwise.
#define DIRT_REF_BAD_ARGS (-1000)
#define DIRT_REF_FRAME_TOO_LARGE (-1001)
//
// With split > 1 the kernel runs split^2 times on the same inputs, each time with grad_pixels kept only on the pixels
// whose (row % split, col % split) is one of the split^2 residues and zero elsewhere, and the outputs of the runs are
// summed in double (grad_vertices64, grad_vertex_colors64).  Every per-pixel term is still the kernel's own fp32
// arithmetic -- a pixel with zero grad_pixels adds exactly zero, and the dilation decisions depend on `pixels` only --
// but each fp32 atomic sum holds 1/split^2 of the terms, so the order-dependent rounding of those sums shrinks by as
// much.  grad_background is exact either way; debug_thingy is that of the first run.
static int assemble(const float* gbuffer, const int32_t* vertex_ids, const float* pixels, const float* grad_pixels,
                    const float* vertices, float* grad_vertices, float* grad_vertex_colors, double* grad_vertices64,
                    double* grad_vertex_colors64, float* grad_background, float* debug_thingy, int B, int H, int W, int C,
                    int V, int split)
{
    if (B <= 0 || H <= 0 || W <= 0 || (C != 1 && C != 3) || V <= 0 || split < 1) return DIRT_REF_BAD_ARGS;
    // framebuffer tiling as in csrc/rasterise_grad_egl.cpp:405-411
    const int horizontal_count = static_cast<int>(std::sqrt(static_cast<float>(B)) + .1f);
    const int vertical_count = B / horizontal_count + (B % horizontal_count == 0 ? 0 : 1);
    const long long buffer_width_ll = (long long)W * horizontal_count, buffer_height_ll = (long long)H * vertical_count;
    // the G-buffer textures are bound as surfaces: a frame the device cannot hold as one is refused before anything
    // is allocated (the reference's GL textures of that size would fail to allocate, csrc/rasterise_grad_egl.cpp:282-314)
    int ordinal = 0, max_surface_w = 0, max_surface_h = 0;
    TRY(cudaGetDevice(&ordinal));
    TRY(cudaDeviceGetAttribute(&max_surface_w, cudaDevAttrMaxSurface2DWidth, ordinal));
    TRY(cudaDeviceGetAttribute(&max_surface_h, cudaDevAttrMaxSurface2DHeight, ordinal));
    if (buffer_width_ll > max_surface_w || buffer_height_ll > max_surface_h) return DIRT_REF_FRAME_TOO_LARGE;
    const int buffer_width = (int)buffer_width_ll, buffer_height = (int)buffer_height_ll;
    const int frames_per_row = buffer_width / W;

    const float inf = std::numeric_limits<float>::infinity();
    std::vector<float4> bary_depth((size_t)buffer_width * buffer_height, make_float4(-1.f, -1.f, -1.f, inf));
    std::vector<float4> indices((size_t)buffer_width * buffer_height, make_float4(-1.f, -1.f, -1.f, -1.f));
    for (int b = 0; b < B; ++b) {
        const int frame_x = (b % frames_per_row) * W, frame_y = (b / frames_per_row) * H;
        for (int r = 0; r < H; ++r)
            for (int c = 0; c < W; ++c) {
                const size_t src = ((size_t)b * H + r) * W + c;
                const size_t dst = (size_t)(frame_y + (H - 1 - r)) * buffer_width + frame_x + c;   // GL rows run bottom-up
                bary_depth[dst] = make_float4(gbuffer[src * 4], gbuffer[src * 4 + 1], gbuffer[src * 4 + 2], gbuffer[src * 4 + 3]);
                // the fragment shader writes a vec3 into an RGBA32F attachment; alpha is never read by assemble_grads
                indices[dst] = make_float4((float)vertex_ids[src * 3], (float)vertex_ids[src * 3 + 1], (float)vertex_ids[src * 3 + 2], 1.f);
            }
    }

    const cudaChannelFormatDesc desc = cudaCreateChannelDesc<float4>();
    DeviceArray bary_array, index_array;
    TRY(cudaMallocArray(&bary_array.a, &desc, buffer_width, buffer_height, cudaArraySurfaceLoadStore));
    TRY(cudaMallocArray(&index_array.a, &desc, buffer_width, buffer_height, cudaArraySurfaceLoadStore));
    const size_t pitch = (size_t)buffer_width * sizeof(float4);
    TRY(cudaMemcpy2DToArray(bary_array.a, 0, 0, bary_depth.data(), pitch, pitch, buffer_height, cudaMemcpyHostToDevice));
    TRY(cudaMemcpy2DToArray(index_array.a, 0, 0, indices.data(), pitch, pitch, buffer_height, cudaMemcpyHostToDevice));

    const size_t n_pix = (size_t)B * H * W;
    DeviceBuffer d_pixels, d_grad_pixels, d_vertices, d_gv, d_gc, d_gb, d_dbg;
    // `pixels` gets 8 zero floats of tail padding: for C = 1 the reference's at() reads "channels" 1 and 2 of the
    // last pixels of the last image past the end of the tensor (csrc/rasterise_grad_egl.cu:119-123); those reads are
    // defined as 0 here, as in the oracle (SURVEY appendix A.4.1)
    TRY(d_pixels.alloc((n_pix * C + 8) * sizeof(float)));
    TRY(cudaMemset(d_pixels.p, 0, (n_pix * C + 8) * sizeof(float)));
    TRY(cudaMemcpy(d_pixels.p, pixels, n_pix * C * sizeof(float), cudaMemcpyHostToDevice));
    // `grad_pixels` gets the same padding: whatever C is, the kernel copies channels 1 and 2 of every pixel into
    // debug_thingy (csrc/rasterise_grad_egl.cu:150-151), which for C = 1 reads up to 8 bytes past the last pixel
    TRY(d_grad_pixels.alloc((n_pix * C + 8) * sizeof(float)));
    TRY(cudaMemset(d_grad_pixels.p, 0, (n_pix * C + 8) * sizeof(float)));
    TRY(d_vertices.alloc((size_t)B * V * 4 * sizeof(float)));
    TRY(cudaMemcpy(d_vertices.p, vertices, (size_t)B * V * 4 * sizeof(float), cudaMemcpyHostToDevice));
    TRY(d_gv.alloc((size_t)B * V * 4 * sizeof(float)));
    TRY(d_gc.alloc((size_t)B * V * C * sizeof(float)));
    TRY(d_gb.alloc(n_pix * C * sizeof(float)));
    TRY(d_dbg.alloc(n_pix * 3 * sizeof(float)));

    tensorflow::Tensor t_gv(d_gv.p, {B, V, 4}), t_gc(d_gc.p, {B, V, C}), t_gb(d_gb.p, {B, H, W, C}), t_dbg(d_dbg.p, {B, H, W, 3});
    const tensorflow::Tensor t_pixels(d_pixels.p, {B, H, W, C}), t_grad_pixels(d_grad_pixels.p, {B, H, W, C}), t_vertices(d_vertices.p, {B, V, 4});
    Eigen::GpuDevice device;
    const cudaArray_t bary_handle = bary_array.a, index_handle = index_array.a;
    const size_t nv4 = (size_t)B * V * 4, nvc = (size_t)B * V * C, ngb = n_pix * C;
    std::vector<float> gp_part, gv_part, gc_part, gb_part;
    if (split > 1) {
        gp_part.resize(ngb); gv_part.resize(nv4); gc_part.resize(nvc); gb_part.resize(ngb);
        std::fill(grad_vertices64, grad_vertices64 + nv4, 0.0);
        std::fill(grad_vertex_colors64, grad_vertex_colors64 + nvc, 0.0);
        std::fill(grad_background, grad_background + ngb, 0.f);
    }
    for (int sy = 0; sy < split; ++sy)
        for (int sx = 0; sx < split; ++sx) {
            const float* gp = grad_pixels;
            if (split > 1) {
                for (size_t p = 0; p < n_pix; ++p) {
                    const bool keep = (int)((p / W) % H) % split == sy && (int)(p % W) % split == sx;
                    for (int ch = 0; ch < C; ++ch) gp_part[p * C + ch] = keep ? grad_pixels[p * C + ch] : 0.f;
                }
                gp = gp_part.data();
            }
            TRY(cudaMemcpy(d_grad_pixels.p, gp, ngb * sizeof(float), cudaMemcpyHostToDevice));
            // the reference's launcher: four memsets, two surface objects, assemble_grads (csrc/rasterise_grad_egl.cu:238-278)
            launch_grad_assembly(t_gv, t_gc, t_gb, t_dbg, bary_handle, index_handle, t_pixels, t_grad_pixels, t_vertices,
                                 buffer_width, buffer_height, device);
            TRY(cudaGetLastError());
            TRY(cudaDeviceSynchronize());
            if (debug_thingy && sy == 0 && sx == 0)
                TRY(cudaMemcpy(debug_thingy, d_dbg.p, n_pix * 3 * sizeof(float), cudaMemcpyDeviceToHost));
            if (split == 1) {
                TRY(cudaMemcpy(grad_vertices, d_gv.p, nv4 * sizeof(float), cudaMemcpyDeviceToHost));
                TRY(cudaMemcpy(grad_vertex_colors, d_gc.p, nvc * sizeof(float), cudaMemcpyDeviceToHost));
                TRY(cudaMemcpy(grad_background, d_gb.p, ngb * sizeof(float), cudaMemcpyDeviceToHost));
                continue;
            }
            TRY(cudaMemcpy(gv_part.data(), d_gv.p, nv4 * sizeof(float), cudaMemcpyDeviceToHost));
            TRY(cudaMemcpy(gc_part.data(), d_gc.p, nvc * sizeof(float), cudaMemcpyDeviceToHost));
            TRY(cudaMemcpy(gb_part.data(), d_gb.p, ngb * sizeof(float), cudaMemcpyDeviceToHost));
            for (size_t i = 0; i < nv4; ++i) grad_vertices64[i] += gv_part[i];
            for (size_t i = 0; i < nvc; ++i) grad_vertex_colors64[i] += gc_part[i];
            for (size_t i = 0; i < ngb; ++i) grad_background[i] += gb_part[i];   // one run writes each pixel, the rest 0
        }
    return 0;
}

extern "C" int dirt_ref_assemble_grads(const float* gbuffer, const int32_t* vertex_ids, const float* pixels,
                                       const float* grad_pixels, const float* vertices, float* grad_vertices,
                                       float* grad_vertex_colors, float* grad_background, float* debug_thingy, int B,
                                       int H, int W, int C, int V)
{
    return assemble(gbuffer, vertex_ids, pixels, grad_pixels, vertices, grad_vertices, grad_vertex_colors, nullptr,
                    nullptr, grad_background, debug_thingy, B, H, W, C, V, 1);
}

// As dirt_ref_assemble_grads, with the vertex gradients summed over split^2 pixel lattices (see assemble) in double.
extern "C" int dirt_ref_assemble_grads_split(const float* gbuffer, const int32_t* vertex_ids, const float* pixels,
                                             const float* grad_pixels, const float* vertices, double* grad_vertices,
                                             double* grad_vertex_colors, float* grad_background, float* debug_thingy,
                                             int B, int H, int W, int C, int V, int split)
{
    if (split < 2) return DIRT_REF_BAD_ARGS;
    return assemble(gbuffer, vertex_ids, pixels, grad_pixels, vertices, nullptr, nullptr, grad_vertices,
                    grad_vertex_colors, grad_background, debug_thingy, B, H, W, C, V, split);
}

// The reference's vertex expansion kernel upload_vertices (csrc/rasterise_grad_egl.cu:12-34) on host arrays:
// expanded [B, 3F] Vertex records (36 bytes each, csrc/rasterise_grad_common.h:5-11).
extern "C" int dirt_ref_upload_vertices(const float* vertices, const int32_t* faces, void* expanded, int B, int V, int F)
{
    if (B <= 0 || V <= 0 || F <= 0) return -1000;
    DeviceBuffer d_vertices, d_faces, d_out;
    TRY(d_vertices.alloc((size_t)B * V * 4 * sizeof(float)));
    TRY(cudaMemcpy(d_vertices.p, vertices, (size_t)B * V * 4 * sizeof(float), cudaMemcpyHostToDevice));
    TRY(d_faces.alloc((size_t)B * F * 3 * sizeof(int32_t)));
    TRY(cudaMemcpy(d_faces.p, faces, (size_t)B * F * 3 * sizeof(int32_t), cudaMemcpyHostToDevice));
    TRY(d_out.alloc((size_t)B * F * 3 * sizeof(Vertex)));
    tensorflow::TTypes<Vertex, 2>::Tensor buffer;
    buffer.data_ = static_cast<Vertex*>(d_out.p);
    buffer.dims_[0] = B; buffer.dims_[1] = (long)F * 3;
    const tensorflow::Tensor t_vertices(d_vertices.p, {B, V, 4}), t_faces(d_faces.p, {B, F, 3});
    Eigen::GpuDevice device;
    launch_vertex_upload(buffer, t_vertices, t_faces, device);
    TRY(cudaGetLastError());
    TRY(cudaDeviceSynchronize());
    TRY(cudaMemcpy(expanded, d_out.p, (size_t)B * F * 3 * sizeof(Vertex), cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int dirt_ref_sizeof_vertex(void) { return (int)sizeof(Vertex); }
