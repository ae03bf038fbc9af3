"""Times the cube-map lookup's CUDA path (dirt_b200.sample_cubemap) against its torch restatement
(tests/cubemap_restatement.py).

    python profiles/cubebench.py [--steps 10] [--rounds 3] [--out FILE]

Workloads: N = 64 x 512^2 lookups, C = 3, into one shared cube map of 6 x 256^2 and one of 6 x 1024^2, for two direction
patterns: `reflection` (each image the reflection vectors of a unit sphere filling it, seen along -z, turned by a
random rotation per image: coherent) and `random` (uniform on the sphere).  For each, alternating op and restatement in
--rounds rounds of --steps calls each (medians over the rounds):
  op_fwd_ms / op_fwd_bwd_ms        the public function through autograd (Python layer and allocations included)
  torch_fwd_ms / torch_fwd_bwd_ms  the restatement in its place
  kernel_fwd_ms                    dirt_cubemap_sample alone on preallocated buffers (the atlas build included)
  border_build_ms                  dirt_cubemap_sample of one lookup: the atlas build, O(6 S^2 C)
  kernel_bwd_ms / kernel_bwd_det_ms  dirt_cubemap_sample_backward, both gradients, default / deterministic
  *_bytes, *_of_peak               algorithmic bytes from shapes / kernel time, against the H100 SXM data sheet's 3.35 TB/s
  op_held_mb / torch_held_mb       device memory autograd holds between forward and backward (output included)
CUDA events on the launching stream.  One JSON object with the card's name and power limit.
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
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from lightbench import PEAK_TBS, card, compare, held_mb, timed  # noqa: E402
import cubemap_restatement as cm  # noqa: E402


def algorithmic_bytes(N, S, C):
    """fwd: read the cube map and write the atlas (the border build), read the directions, write the output.
    bwd: read directions and grad_out, write grad_directions; zero, then read the atlas gradient, and write grad_cubemap.
    Texel reads by the lookups are counted once, as the cube map's size."""
    cube, atlas = 4 * 6 * S * S * C, 4 * 6 * (S + 2) ** 2 * C
    return cube + 2 * atlas + 4 * N * (3 + C), 4 * N * (3 + C + 3) + 2 * atlas + cube


def directions(pattern, B, H, W, dev, g):
    if pattern == 'random':
        return torch.randn(B, H * W, 3, generator=g, device=dev)
    ys, xs = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing='ij')
    x, y = (xs + 0.5) / W * 2 - 1, 1 - (ys + 0.5) / H * 2
    r2 = x * x + y * y
    n = torch.stack([x, y, torch.sqrt((1 - r2).clamp_min(0))], -1)
    v = torch.tensor([0., 0., -1.], device=dev)
    refl = v - 2 * (n * v).sum(-1, keepdim=True) * n
    refl = torch.where((r2 < 1)[..., None], refl, torch.stack([x, y, -torch.ones_like(x)], -1)).reshape(1, H * W, 3)
    q = torch.nn.functional.normalize(torch.randn(B, 4, generator=g, device=dev), dim=-1)   # per-image rotation
    a, b, c, d = q.unbind(-1)
    R = torch.stack([1 - 2 * (c * c + d * d), 2 * (b * c - a * d), 2 * (b * d + a * c),
                     2 * (b * c + a * d), 1 - 2 * (b * b + d * d), 2 * (c * d - a * b),
                     2 * (b * d - a * c), 2 * (c * d + a * b), 1 - 2 * (b * b + c * c)], -1).reshape(B, 3, 3)
    return (refl @ R).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('cubebench.py needs a CUDA device')
    import dirt_b200 as dirt
    from dirt_b200 import _lib
    L = _lib.lib()
    dev = torch.device('cuda', 0)
    B, H, W, C = 64, 512, 512, 3
    N = H * W
    name, limit = card()
    result = {'device': name, 'power_limit': limit, 'lookups': B * N, 'channels': C, 'steps': args.steps,
              'rounds': args.rounds, 'cases': []}
    g = torch.Generator(device=dev).manual_seed(0)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    grad_out = torch.randn(B, N, C, generator=g, device=dev)
    for S in (256, 1024):
        cube = torch.rand(6, S, S, C, generator=g, device=dev)
        cm.border_table(S)   # built once per size, outside the timed window
        for pattern in ('reflection', 'random'):
            dirs = directions(pattern, B, H, W, dev, g)
            leaves = [cube.clone().requires_grad_(True), dirs.clone().requires_grad_(True)]

            def fwd(fn):
                with torch.no_grad():
                    return fn(cube, dirs)

            def fwd_bwd(fn):
                for v in leaves:
                    v.grad = None
                fn(*leaves).backward(grad_out)

            atlas = torch.empty(int(L.dirt_cubemap_atlas_bytes(1, S, C)) // 4, device=dev)
            out = torch.empty(B, N, C, device=dev)
            gc, gd = torch.empty_like(cube), torch.empty_like(dirs)
            scratch = {det: torch.empty(int(L.dirt_cubemap_sample_backward_bytes(1, S, C, B, N, 0, det)),
                                        dtype=torch.uint8, device=dev) for det in (0, 1)}
            run_fwd = lambda: L.dirt_cubemap_sample(p(cube), p(dirs), p(atlas), p(out), 1, S, C, B, N, 0, stream())
            run_build = lambda: L.dirt_cubemap_sample(p(cube), p(dirs), p(atlas), p(out), 1, S, C, 1, 1, 0, stream())
            run_bwd = {det: (lambda det=det: L.dirt_cubemap_sample_backward(
                p(atlas), p(dirs), p(grad_out), p(gc), p(gd), 1, S, C, B, N, 0, det, p(scratch[det]),
                scratch[det].numel(), stream())) for det in (0, 1)}
            assert run_fwd() == 0
            times = ([], [], [], [])
            for _ in range(args.rounds):
                for t, fn in zip(times, (run_fwd, run_build, run_bwd[0], run_bwd[1])):
                    t.append(timed(fn, args.steps))
            k_fwd, k_build, k_bwd, k_det = (statistics.median(t) for t in times)
            op_fwd, torch_fwd = compare(lambda: fwd(dirt.sample_cubemap), lambda: fwd(cm.sample), args.steps, args.rounds)
            op_fb, torch_fb = compare(lambda: fwd_bwd(dirt.sample_cubemap), lambda: fwd_bwd(cm.sample), args.steps,
                                      args.rounds)
            fb, bb = algorithmic_bytes(B * N, S, C)
            row = {'case': '%s, 6 x %d^2' % (pattern, S), 'op_fwd_ms': op_fwd, 'torch_fwd_ms': torch_fwd,
                   'op_fwd_bwd_ms': op_fb, 'torch_fwd_bwd_ms': torch_fb, 'kernel_fwd_ms': k_fwd,
                   'border_build_ms': k_build, 'kernel_bwd_ms': k_bwd, 'kernel_bwd_det_ms': k_det,
                   'fwd_bytes': fb, 'bwd_bytes': bb,
                   'kernel_fwd_of_peak': fb / (k_fwd * 1e-3) / 1e12 / PEAK_TBS,
                   'kernel_bwd_of_peak': bb / (k_bwd * 1e-3) / 1e12 / PEAK_TBS,
                   'op_held_mb': held_mb(lambda: dirt.sample_cubemap(*leaves)),
                   'torch_held_mb': held_mb(lambda: cm.sample(*leaves)),
                   'speedup_fwd': torch_fwd / op_fwd, 'speedup_fwd_bwd': torch_fb / op_fb}
            result['cases'].append(row)
            print(json.dumps(row), flush=True)
            del leaves, atlas, out, gc, gd, scratch, dirs
            torch.cuda.empty_cache()
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            f.write(json.dumps(result, indent=1) + '\n')


if __name__ == '__main__':
    main()
