"""Times sample_texture(mode='trilinear') against its torch restatement and against mode='bilinear'.

    python profiles/mipbench.py [--steps 20] [--out FILE]

Workload: texbench's, N = 64 x 512^2 lookups, C = 3, one shared 1024^2 texture.  The `gbuffer` pattern is scaled about
each image's origin so that the median footprint from index_derivatives is rho = 1, 4 and 16 texels per pixel; `random`
is uniform over the texture.  The derivatives come from index_derivatives of the index image.  For each case:
  op_fwd_ms / op_fwd_bwd_ms           sample_texture(mode='trilinear') through autograd (pyramid build included)
  restatement_fwd_ms / _fwd_bwd_ms    tests/texture_mip_restatement.py's sample in float32, same calls
  bilinear_fwd_ms / _fwd_bwd_ms       sample_texture(mode='bilinear') on the same indices
  build_ms, helper_ms                 dirt_texture_mip_build alone; index_derivatives alone
  kernel_fwd_ms, kernel_bwd_ms        the C ABI alone on preallocated buffers (backward: both gradients, memsets and the
                                      collapse included); kernel_bwd_det_ms the same call with deterministic = 1
  *_tbs                               algorithmic bytes / kernel time, against the H100 SXM data sheet's 3.35 TB/s
CUDA events on the launching stream, averaged over --steps calls after warm-up (the restatement: 3 calls).  One JSON
object with the card's name and power limit, read in the same run.
"""
import argparse
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from texbench import PEAK_TBS, card, gbuffer_indices, timed  # noqa: E402


def algorithmic_bytes(N, texels, C):
    """fwd: read the index pair, the 4 derivatives, write C floats per lookup; read level 0 and the pyramid (4/3 of the
    texture) once.  bwd: per lookup read the index pair, the derivatives and C floats of grad_out, write the index
    gradient; read the texture and pyramid once (index gradient), zero and write the per-level gradients once each,
    read them once in the collapse and write grad_texture."""
    levels = texels * 4 * C * 4 / 3
    fwd = N * (8 + 16 + 4 * C) + levels
    bwd = N * (8 + 16 + 4 * C + 8) + 3 * levels + texels * 4 * C
    return fwd, bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import dirt_b200 as dirt
    from dirt_b200 import _lib
    import texture_mip_restatement as mip
    L = _lib.lib()
    dev = torch.device('cuda', 0)
    B, H, W, C, size = 64, 512, 512, 3, 1024
    N = B * H * W
    name, limit = card()
    result = {'device': name, 'power_limit': limit, 'lookups': N, 'channels': C, 'texture': size, 'steps': args.steps,
              'cases': []}
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    texture = torch.rand(size, size, C, device=dev)
    pyramid = torch.empty(L.dirt_texture_mip_pyramid_bytes(1, size, size, C) // 4, device=dev)
    base = gbuffer_indices(B, H, W, size, dev).reshape(B, H * W, 2)
    rho0 = float(dirt.index_derivatives(base.reshape(B, H, W, 2), (size, size)).reshape(-1, 2, 2).norm(dim=-1).amax(-1).median())
    for pattern, rho in (('gbuffer', 1), ('gbuffer', 4), ('gbuffer', 16), ('random', None)):
        if pattern == 'gbuffer':
            origin = base[:, :1]
            indices = ((base - origin) * (rho / rho0) + origin).reshape(-1, 2).contiguous()
        else:
            indices = (torch.rand(N, 2, device=dev) * size).contiguous()
        image = indices.reshape(B, H, W, 2)
        derivatives = dirt.index_derivatives(image, (size, size)).reshape(N, 4).contiguous()
        lam = mip.lod(derivatives, mip.level_count(size, size))
        grad_out = torch.randn(N, C, device=dev)
        out = torch.empty(N, C, device=dev)
        grad_texture = torch.empty_like(texture)
        grad_indices = torch.empty_like(indices)
        assert L.dirt_texture_mip_build(p(texture), p(pyramid), 1, size, size, C, stream()) == 0
        sizes = {d: int(L.dirt_texture_sample_trilinear_backward_bytes(1, size, size, C, 1, N, d)) for d in (0, 1)}
        scratch = {d: torch.empty(sizes[d], dtype=torch.uint8, device=dev) for d in (0, 1)}

        def k_bwd(det):
            return L.dirt_texture_sample_trilinear_backward(p(texture), p(pyramid), p(indices), p(derivatives), p(grad_out),
                                                            p(grad_texture), p(grad_indices), 1, size, size, C, 1, N, det,
                                                            p(scratch[det]), sizes[det], stream())

        k_fwd = timed(lambda: L.dirt_texture_sample_trilinear(p(texture), p(pyramid), p(indices), p(derivatives), p(out), 1,
                                                              size, size, C, 1, N, stream()), args.steps)
        k_build = timed(lambda: L.dirt_texture_mip_build(p(texture), p(pyramid), 1, size, size, C, stream()), args.steps)
        k_b = timed(lambda: k_bwd(0), args.steps)
        k_d = timed(lambda: k_bwd(1), max(3, args.steps // 4))
        helper = timed(lambda: dirt.index_derivatives(image, (size, size)), args.steps)
        tex_p, idx_p = texture.clone().requires_grad_(True), indices.clone().requires_grad_(True)

        def fwd(fn):
            with torch.no_grad():
                fn(texture, indices)

        def fwd_bwd(fn):
            tex_p.grad, idx_p.grad = None, None
            fn(tex_p, idx_p).backward(grad_out)

        tri = lambda t, i: dirt.sample_texture(t, i, mode='trilinear', derivatives=derivatives)
        bil = lambda t, i: dirt.sample_texture(t, i, mode='bilinear')
        ref = lambda t, i: mip.sample(t, i, derivatives)
        fb, bb = algorithmic_bytes(N, size * size, C)
        case = {'pattern': pattern, 'rho_target': rho,
                'lambda_median': float(lam[0].add(lam[1]).median()),
                'op_fwd_ms': timed(lambda: fwd(tri), args.steps),
                'op_fwd_bwd_ms': timed(lambda: fwd_bwd(tri), args.steps),
                'restatement_fwd_ms': timed(lambda: fwd(ref), 3, warmup=1),
                'restatement_fwd_bwd_ms': timed(lambda: fwd_bwd(ref), 3, warmup=1),
                'bilinear_fwd_ms': timed(lambda: fwd(bil), args.steps),
                'bilinear_fwd_bwd_ms': timed(lambda: fwd_bwd(bil), args.steps),
                'build_ms': k_build, 'helper_ms': helper,
                'kernel_fwd_ms': k_fwd, 'kernel_bwd_ms': k_b, 'kernel_bwd_det_ms': k_d,
                'det_over_default': k_d / k_b,
                'scratch_bytes_default': sizes[0], 'scratch_bytes_det': sizes[1],
                'fwd_bytes': fb, 'bwd_bytes': bb,
                'fwd_tbs': fb / (k_fwd * 1e-3) / 1e12, 'bwd_tbs': bb / (k_b * 1e-3) / 1e12}
        case['fwd_of_peak'] = case['fwd_tbs'] / PEAK_TBS
        case['bwd_of_peak'] = case['bwd_tbs'] / PEAK_TBS
        result['cases'].append(case)
        print(json.dumps(case), flush=True)
        del scratch
        torch.cuda.empty_cache()
    text = json.dumps(result, indent=1)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(text + '\n')
    print(text)


if __name__ == '__main__':
    main()
