"""Times the spherical-harmonics lighting's CUDA path against its torch restatement (dirt_b200/lighting.py).

    python profiles/shbench.py [--steps 20] [--rounds 3] [--out FILE] [--variant TAG=LIB ...]

Workloads: the op alone on N = 64 x 512^2 points, C = 3, contiguous inputs, with shared and with per-item
coefficients; and a deferred shader (albedo * SH, blended with a background colour by the mask) on a 64 x 512 x 512 x 7
G-buffer [mask, albedo rgb, normal xyz] with per-item coefficients (its per-point inputs are strided slices).  For each,
alternating op and restatement in --rounds rounds of --steps calls each (the figures are medians over the rounds):
  op_fwd_ms / op_fwd_bwd_ms        the public function through autograd (Python layer and allocations included)
  torch_fwd_ms / torch_fwd_bwd_ms  the same call with the restatement in its place
  kernel_fwd_ms / kernel_bwd_ms    the C ABI alone on preallocated buffers (backward: every gradient, the reduction
                                   kernel included); kernel_bwd_coef_only_ms: only the coefficient gradient
  *_bytes, *_of_peak               algorithmic bytes from shapes / kernel time, against the H100 SXM data sheet's 3.35 TB/s
  op_held_mb / torch_held_mb       device memory autograd holds between forward and backward (output included)
--variant TAG=LIB times the same ABI calls on another build of the library (profiles/build_variant.py), alternating
with the product build, e.g. to compare points per thread of the backward kernel.  CUDA events on the launching
stream.  One JSON object with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))
from lightbench import PEAK_TBS, card, compare, held_mb, timed  # noqa: E402


def algorithmic_bytes(N, C):
    """fwd: read normals and albedo once, write the output.  bwd: read normals, albedo and grad_out, write grad_normals
    and grad_albedo (the coefficients, their gradient and the partials are negligible)."""
    return 4 * N * (3 + 2 * C), 4 * N * (3 + 2 * C + 3 + C)


def restatement(lighting):
    def fn(vertex_normals, vertex_colors, coefficients, name=None):
        return lighting._diffuse_spherical_harmonics(vertex_normals, vertex_colors, coefficients)
    return fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    ap.add_argument('--variant', action='append', default=[])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('shbench.py needs a CUDA device')
    from dirt_b200 import _lib, lighting
    libs = {'product': _lib.lib()}
    for spec in args.variant:
        tag, path = spec.split('=', 1)
        libs[tag] = _lib.load(path)
    dev = torch.device('cuda', 0)
    B, H, W, C = 64, 512, 512, 3
    N = H * W
    name, limit = card()
    result = {'device': name, 'power_limit': limit, 'points': B * N, 'channels': C, 'steps': args.steps,
              'rounds': args.rounds, 'cases': []}
    g = torch.Generator(device=dev).manual_seed(0)
    nrm = torch.nn.functional.normalize(torch.randn(B, N, 3, generator=g, device=dev), dim=-1)
    alb = torch.rand(B, N, C, generator=g, device=dev)
    coef_item = torch.randn(B, 9, C, generator=g, device=dev) * 0.3
    coef_item[:, 0] += 3.
    grad_out = torch.randn(B, N, C, generator=g, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    op_fn, ref_fn = lighting.diffuse_spherical_harmonics, restatement(lighting)
    fb, bb = algorithmic_bytes(B * N, C)
    for case, coef in (('op alone, shared coefficients', coef_item[0].contiguous()),
                       ('op alone, per-item coefficients', coef_item)):
        per_item = coef.dim() == 3
        leaves = [t.clone().requires_grad_(True) for t in (nrm, alb, coef)]

        def fwd(fn):
            with torch.no_grad():
                return fn(nrm, alb, coef)

        def fwd_bwd(fn):
            for v in leaves:
                v.grad = None
            fn(*leaves).backward(grad_out)

        out = torch.empty(B, N, C, device=dev)
        grads = [torch.empty(B, N, 3, device=dev), torch.empty(B, N, C, device=dev), torch.empty_like(coef)]
        inputs = [p(nrm), 3, p(alb), C, p(coef), int(per_item)]
        def abi_calls(L):
            ws_bytes = int(L.dirt_sh_lighting_workspace_bytes(B, N, C))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            run_fwd = lambda: L.dirt_sh_lighting_forward(*inputs, p(out), B, N, C, stream())
            run_bwd = lambda: L.dirt_sh_lighting_backward(*inputs, p(grad_out), *[p(t) for t in grads], p(ws), ws_bytes,
                                                          B, N, C, stream())
            run_coef = lambda: L.dirt_sh_lighting_backward(*inputs, p(grad_out), p(None), p(None), p(grads[2]), p(ws),
                                                           ws_bytes, B, N, C, stream())
            return run_fwd, run_bwd, run_coef

        kernels = {tag: abi_calls(L) for tag, L in libs.items()}
        times = {tag: ([], [], []) for tag in libs}
        for _ in range(args.rounds):
            for tag, fns in kernels.items():
                for t, fn in zip(times[tag], fns):
                    t.append(timed(fn, args.steps))
        k_fwd, k_bwd, k_coef = (statistics.median(t) for t in times['product'])
        op_fwd, torch_fwd = compare(lambda: fwd(op_fn), lambda: fwd(ref_fn), args.steps, args.rounds)
        op_fb, torch_fb = compare(lambda: fwd_bwd(op_fn), lambda: fwd_bwd(ref_fn), args.steps, args.rounds)
        row = {'case': case, 'op_fwd_ms': op_fwd, 'torch_fwd_ms': torch_fwd, 'op_fwd_bwd_ms': op_fb,
               'torch_fwd_bwd_ms': torch_fb, 'kernel_fwd_ms': k_fwd, 'kernel_bwd_ms': k_bwd,
               'kernel_bwd_coef_only_ms': k_coef, 'fwd_bytes': fb, 'bwd_bytes': bb,
               'kernel_fwd_of_peak': fb / (k_fwd * 1e-3) / 1e12 / PEAK_TBS,
               'kernel_bwd_of_peak': bb / (k_bwd * 1e-3) / 1e12 / PEAK_TBS,
               'op_held_mb': held_mb(lambda: op_fn(*leaves)), 'torch_held_mb': held_mb(lambda: ref_fn(*leaves))}
        row['speedup_fwd'] = torch_fwd / op_fwd
        row['speedup_fwd_bwd'] = torch_fb / op_fb
        for tag in libs:
            if tag != 'product':
                row['variant_' + tag] = dict(zip(('kernel_fwd_ms', 'kernel_bwd_ms', 'kernel_bwd_coef_only_ms'),
                                                 (statistics.median(t) for t in times[tag])))
        result['cases'].append(row)
        print(json.dumps(row), flush=True)
        del leaves, out, grads, kernels
        torch.cuda.empty_cache()

    # a deferred shader on a cfg3-sized G-buffer: albedo * SH, blended with the background by the mask
    del nrm, alb, grad_out
    torch.cuda.empty_cache()
    gbuffer = torch.rand(B, H, W, 7, generator=g, device=dev)
    gbuffer[..., 0] = (gbuffer[..., 0] > 0.2).float()
    gbuffer[..., 4:] = torch.nn.functional.normalize(gbuffer[..., 4:] - 0.5, dim=-1)
    bg_colour = torch.tensor([0.1, 0.2, 0.3], device=dev)
    shade_grad = torch.randn(B, H, W, 3, generator=g, device=dev)
    gb = gbuffer.clone().requires_grad_(True)
    cf = coef_item.clone().requires_grad_(True)

    def shader(sh, gbuf, coefficients):
        mask, albedo, normals = gbuf[..., :1], gbuf[..., 1:4], gbuf[..., 4:7]
        lit = sh(normals.reshape(B, -1, 3), albedo.reshape(B, -1, 3), coefficients).reshape(B, H, W, 3)
        return lit * mask + bg_colour * (1. - mask)

    def shader_fwd(sh):
        with torch.no_grad():
            return shader(sh, gbuffer, coef_item)

    def shader_fwd_bwd(sh):
        gb.grad, cf.grad = None, None
        shader(sh, gb, cf).backward(shade_grad)

    op_fwd, torch_fwd = compare(lambda: shader_fwd(op_fn), lambda: shader_fwd(ref_fn), args.steps, args.rounds)
    op_fb, torch_fb = compare(lambda: shader_fwd_bwd(op_fn), lambda: shader_fwd_bwd(ref_fn), args.steps, args.rounds)
    row = {'case': 'deferred shader, per-item coefficients', 'op_fwd_ms': op_fwd, 'torch_fwd_ms': torch_fwd,
           'op_fwd_bwd_ms': op_fb, 'torch_fwd_bwd_ms': torch_fb,
           'op_held_mb': held_mb(lambda: shader(op_fn, gb, cf)), 'torch_held_mb': held_mb(lambda: shader(ref_fn, gb, cf)),
           'speedup_fwd': torch_fwd / op_fwd, 'speedup_fwd_bwd': torch_fb / op_fb}
    result['cases'].append(row)
    print(json.dumps(row), flush=True)
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            f.write(json.dumps(result, indent=1) + '\n')


if __name__ == '__main__':
    main()
