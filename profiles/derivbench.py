"""Times the G-buffer derivative kernel (DESIGN.md §7.7) against index_derivatives, alone and inside a textured
deferred pipeline.

    python profiles/derivbench.py [--steps 20] [--out FILE]

Workload: cfg3's geometry (64 x 512^2, icosphere-4, per-item pose) with spherical uv added as G-buffer channels 4, 5
(u = atan2(nz, nx) / 2pi + 0.5, v = acos(ny) / pi of the posed unit normal; the faces across u = 0 / 1 are a seam), C = 6,
and a 1024^2 texture of 3 channels.  Reported:
  kernel_ms                 dirt_rasterise_derivatives of the two uv channels alone, on the forward call's workspace
  kernel_bytes, kernel_tbs  B*H*W*(4 + 8K) (face id in, 2K floats out) plus every face's 64-byte record and three
                            K-float attribute rows read once, over kernel time, against the H100 SXM data sheet's 3.35 TB/s
  helper_ms                 index_derivatives of the same pixels' texel indices
  pipeline_analytic_ms      rasterise_batch_deferred with derivative_channels=range(4, 6), a shader doing
                            sample_texture(mode='trilinear'), and the backward pass to the texture
  pipeline_helper_ms        the same with the derivatives from index_derivatives of the G-buffer's indices
  level_differs             fraction of covered pixels where the two routes give a different floor(lambda)
CUDA events on the launching stream, averaged over --steps calls after warm-up.  One JSON object with the card's name
and power limit, read in the same run.
"""
import argparse
import ctypes
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from texbench import PEAK_TBS, card, timed  # noqa: E402


def scene_with_uv(dev):
    from dirt_b200 import scenes
    s = scenes.config3()
    t = {k: torch.from_numpy(v).to(dev) for k, v in s.items()}
    n = t['vertex_colors'][..., 1:4]
    u = torch.atan2(n[..., 2], n[..., 0]) / (2 * math.pi) + 0.5
    v = torch.acos(n[..., 1].clamp(-1., 1.)) / math.pi
    t['vertex_colors'] = torch.cat([t['vertex_colors'], u[..., None], v[..., None]], -1).contiguous()
    t['background'] = torch.zeros(t['background'].shape[:3] + (6,), device=dev)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import dirt_b200 as dirt
    from dirt_b200 import _lib, rasterise_ops
    import texture_mip_restatement as mip
    L = _lib.lib()
    dev = torch.device('cuda', 0)
    name, limit = card()
    t = scene_with_uv(dev)
    B, H, W, C = t['background'].shape
    V, F = t['vertices'].shape[1], t['faces'].shape[1]
    K, size = 2, 1024
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

    gbuffer, ids, ws = rasterise_ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'],
                                                           return_workspace=True)
    out = torch.empty(B, H, W, 2, K, device=dev)

    def kernel():
        rc = L.dirt_rasterise_derivatives(p(t['vertices']), p(t['faces']), p(t['vertex_colors']), p(ids), p(out), B, H, W, C,
                                          V, F, 4, K, 1, p(ws), ws.numel(), stream())
        assert rc == 0, rc

    kernel_ms = timed(kernel, args.steps)
    covered = int((ids >= 0).sum())
    kernel_bytes = B * H * W * (4 + 8 * K) + B * F * (64 + 3 * 4 * K)
    indices = dirt.uvs_to_pixel_indices(gbuffer[..., 4:6], (size, size))
    helper = lambda: dirt.index_derivatives(indices, (size, size))
    helper_ms = timed(helper, args.steps)

    scale = torch.tensor([float(size), float(size)], device=dev)
    analytic = (out.flip(-1) * scale).flatten(-2)
    levels = mip.level_count(size, size)
    cov = ids >= 0
    level_differs = float((mip.lod(analytic, levels)[0] != mip.lod(helper(), levels)[0])[..., 0][cov].float().mean())

    texture = torch.rand(size, size, 3, device=dev).requires_grad_(True)
    grad_out = torch.randn(B, H, W, 3, device=dev)

    def shader_analytic(g, tex, gbuffer_derivatives):
        d = (gbuffer_derivatives.flip(-1) * scale).flatten(-2)
        return dirt.sample_texture(tex, dirt.uvs_to_pixel_indices(g[..., 4:6], (size, size)), mode='trilinear', derivatives=d)

    def shader_helper(g, tex):
        idx = dirt.uvs_to_pixel_indices(g[..., 4:6], (size, size))
        return dirt.sample_texture(tex, idx, mode='trilinear', derivatives=dirt.index_derivatives(idx, (size, size)))

    def pipeline(shader, **kw):
        texture.grad = None
        px = dirt.rasterise_batch_deferred(t['background'], t['vertices'], t['vertex_colors'], t['faces'], shader, [texture],
                                           **kw)
        px.backward(grad_out)

    result = {'device': name, 'power_limit': limit, 'batch': B, 'height': H, 'width': W, 'channels': C,
              'derivative_channels': K, 'texture': size, 'steps': args.steps, 'covered_pixels': covered,
              'kernel_ms': kernel_ms, 'kernel_bytes': kernel_bytes,
              'kernel_tbs': kernel_bytes / (kernel_ms * 1e-3) / 1e12,
              'helper_ms': helper_ms,
              'pipeline_analytic_ms': timed(lambda: pipeline(shader_analytic, derivative_channels=range(4, 6)), args.steps),
              'pipeline_helper_ms': timed(lambda: pipeline(shader_helper), args.steps),
              'level_differs': level_differs}
    result['kernel_of_peak'] = result['kernel_tbs'] / PEAK_TBS
    result['helper_over_kernel'] = helper_ms / kernel_ms
    text = json.dumps(result, indent=1)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(text + '\n')
    print(text)


if __name__ == '__main__':
    main()
