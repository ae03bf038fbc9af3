// grad_pixel.cuh -- the per-pixel decisions of the RasteriseGrad pass that both backward paths make: the Scharr sums of
// a channel group read from global memory and the occluder-edge dilation of assemble_grads
// (csrc/rasterise_grad_egl.cu:126-127, 155-194).  backward.cu's reference-shaped tile path and deterministic.cu's record
// pass call the same inline code, so the deterministic path takes every decision the default path takes.
#pragma once
#include "common.cuh"

namespace dirt {

struct V3 { float x, y, z; };

// at(): nearest frame pixel for out-of-range taps; three components of the channel group starting at
// c0 (width n).  For n == 1 the reference reads "channels" 1 and 2 of a contiguous [B,H,W,1] tensor,
// i.e. the next two pixels in flat order (0 past the end of the tensor).
struct Frame { int B, H, W; };
__device__ __forceinline__ V3 group_at(const float* __restrict__ pixels, int b, int r, int c, const Frame d, int cs, int c0, int n)
{
    r = max(0, min(d.H - 1, r));
    c = max(0, min(d.W - 1, c));
    const size_t lin = ((size_t)b * d.H + r) * d.W + c;
    V3 v;
    if (n == 3) {
        const float* p = pixels + lin * cs + c0;
        v.x = __ldg(p); v.y = __ldg(p + 1); v.z = __ldg(p + 2);
    } else {
        const size_t total = (size_t)d.B * d.H * d.W;
        v.x = __ldg(pixels + lin * cs + c0);
        v.y = (lin + 1 < total) ? __ldg(pixels + (lin + 1) * cs + c0) : 0.f;
        v.z = (lin + 2 < total) ? __ldg(pixels + (lin + 2) * cs + c0) : 0.f;
    }
    return v;
}

// (a + b - c - d) * 3/32 + (e - f) * 10/32 in the order of operations of the reference's compiled kernel
// (csrc/rasterise_grad_egl.cu:126-127 as nvcc contracts it: FMUL (e-f)*10/32, then FFMA (a+b-c-d)*3/32 + that; the SASS of
// oracle/_ref, `make -C oracle ref-sass`)
__device__ __forceinline__ float scharr_comp(float a, float b, float c, float dd, float e, float f)
{
    const float X = __fsub_rn(__fsub_rn(__fadd_rn(a, b), c), dd);
    const float Y = __fsub_rn(e, f);
    return __fmaf_rn(X, 0.09375f, __fmul_rn(Y, 0.3125f));
}

__device__ __forceinline__ float l1(const float s[3])
{
    return __fadd_rn(__fadd_rn(fabsf(s[0]), fabsf(s[1])), fabsf(s[2]));
}

// global-memory taps (tiles at the right frame edge, where the flat-order reads of a 1-wide group wrap into the next
// row): three components of group [c0, c0+N0) at the clamped pixel
template <int N0>
__device__ __forceinline__ void scharr_global(const float* __restrict__ pixels, int b, int row, int col, const Frame d, int cs,
                                              int c0, float (&sx)[3], float (&sy)[3])
{
    const V3 a_mm = group_at(pixels, b, row + 1, col - 1, d, cs, c0, N0), a_mp = group_at(pixels, b, row - 1, col - 1, d, cs, c0, N0);
    const V3 a_pm = group_at(pixels, b, row + 1, col + 1, d, cs, c0, N0), a_pp = group_at(pixels, b, row - 1, col + 1, d, cs, c0, N0);
    const V3 a_m0 = group_at(pixels, b, row, col - 1, d, cs, c0, N0), a_p0 = group_at(pixels, b, row, col + 1, d, cs, c0, N0);
    const V3 a_0m = group_at(pixels, b, row + 1, col, d, cs, c0, N0), a_0p = group_at(pixels, b, row - 1, col, d, cs, c0, N0);
    sx[0] = scharr_comp(a_mm.x, a_mp.x, a_pm.x, a_pp.x, a_m0.x, a_p0.x);
    sx[1] = scharr_comp(a_mm.y, a_mp.y, a_pm.y, a_pp.y, a_m0.y, a_p0.y);
    sx[2] = scharr_comp(a_mm.z, a_mp.z, a_pm.z, a_pp.z, a_m0.z, a_p0.z);
    sy[0] = scharr_comp(a_mm.x, a_pm.x, a_mp.x, a_pp.x, a_0m.x, a_0p.x);
    sy[1] = scharr_comp(a_mm.y, a_pm.y, a_mp.y, a_pp.y, a_0m.y, a_0p.y);
    sy[2] = scharr_comp(a_mm.z, a_pm.z, a_mp.z, a_pp.z, a_0m.z, a_0p.z);
}

// Dilation codes (the record planes of dirt_rasterise_backward_deterministic, include/dirt_b200.h): bits 0-1 say which
// fragment receives the pixel's position gradient, bit 2 that the preferred step runs along the row.
constexpr int DIL_NONE = 0, DIL_OWN = 1, DIL_FIRST = 2, DIL_SECOND = 3, DIL_ALONG_ROW = 4;

// The dilation of assemble_grads (:155-194) at an interior pixel (col, row) whose own face is f_own (record t_own,
// G-buffer entry g_own): the neighbour one step along the dominant Scharr axis (dithered by (col+row)%2), else the one
// opposite, takes over the pixel's position gradient if it is covered, shows a different triangle (vertex triple) and is
// nearer.  On a take-over f, g and tf become the neighbour's face id, its G-buffer entry AT THE NEIGHBOUR and its record.
// `ids` is the image's face-id plane.  `code` receives DIL_OWN, DIL_FIRST or DIL_SECOND, with DIL_ALONG_ROW when the
// preferred step runs along the row (callers that only need f, g and tf ignore it).
__device__ __forceinline__ void dilate_generic(const int32_t* ids, const TriInterp* __restrict__ itp_b, const Frame d, int col,
                                               int row, const float (&sx)[3], const float (&sy)[3], int f_own,
                                               const TriInterp& t_own, const float4& g_own, int& f, float4& g, TriInterp& tf,
                                               int& code)
{
    int dx = (l1(sx) > l1(sy)) ? 1 : 0, dy = 1 - dx;  // buffer (y-up) orientation
    code = dx ? (DIL_ALONG_ROW | DIL_OWN) : DIL_OWN;
    if ((col + row) & 1) { dx = -dx; dy = -dy; }
    for (int attempt = 0; attempt < 2; ++attempt) {
        const int nc = col + dx, nr = row - dy;
        const int fn = ids[nr * d.W + nc];
        if (fn >= 0) {
            const TriInterp tn = load_interp(itp_b + fn);
            const bool differs = (f_own < 0) || tn.v0 != t_own.v0 || tn.v1 != t_own.v1 || tn.v2 != t_own.v2;
            const float4 gn = exact::gbuffer_at(tn, nc, nr);
            if (differs && g_own.w > gn.w) {
                g = gn; f = fn; tf = tn;
                code += 1 + attempt;
                break;
            }
        }
        dx = -dx; dy = -dy;
    }
}

}  // namespace dirt
