"""Times vertex_tangents and perturb_normals (dirt_b200/lighting.py, DESIGN.md §7.14) against their torch restatements.

    python profiles/normalmapbench.py [--steps 20] [--rounds 3] [--out FILE]

Workloads:
  a  vertex_tangents, cfg5-sized seamed uv sphere (224 x 112, V = 25425, F = 49952), B = 64 per-item positions, shared uvs
  b  vertex_tangents, seamed uv sphere 1024 x 512 (V = 525825), B = 1
  c  perturb_normals, 64 x 512^2 points, contiguous [64, 512^2, k] inputs
  d  perturb_normals, the same points as views of a [64, 512, 512, 14] G-buffer (normal, tangent, sample channels)
For each, alternating op and restatement in --rounds rounds of --steps calls each (medians over the rounds):
  op_fwd_ms / op_fwd_bwd_ms        the public function through autograd (Python layer and allocations included)
  torch_fwd_ms / torch_fwd_bwd_ms  the same call with the restatement in its place
  kernel_fwd_ms / kernel_bwd_ms    the C ABI alone on preallocated buffers (the tangents' forward includes the adjacency)
  *_launches                       kernels and memsets per call (the C ABI's count; torch.profiler for fwd + bwd)
  *_bytes, *_of_peak               algorithmic bytes from shapes / kernel time, against the H100 SXM data sheet's 3.35 TB/s
  op_held_mb / torch_held_mb       device memory autograd holds between forward and backward (output included)
CUDA events on the launching stream.  One JSON object with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'examples'))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lightbench import PEAK_TBS, card, compare, held_mb, timed   # noqa: E402
from normalmap import seamed_sphere   # noqa: E402


def tangent_bytes(B, V, F):
    """fwd: read the faces, each item's positions and normals once and the shared uvs, write [B*V, 4].  bwd: read the
    faces, positions, uvs, normals and grad_tangents; write and read the per-vertex gradient; write the vertex, uv and
    normal gradients."""
    fwd = 12 * F + 8 * V + B * V * (12 + 12 + 16)
    bwd = 12 * F + 8 * V + B * V * (12 + 12 + 16 + 2 * 12 + 12 + 8 + 12)
    return fwd, bwd


def perturb_bytes(N):
    """fwd: read 3 + 4 + 3 floats per point, write 3.  bwd: read those and grad_out, write 3 + 4 + 3."""
    return N * 4 * 13, N * 4 * 23


def profile_launches(fn, steps=5):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA) / steps


def tangent_case(label, columns, rows, B, args, L, lighting, dev):
    p, uv, faces = seamed_sphere(columns, rows, dev)
    g = torch.Generator(device=dev).manual_seed(0)
    V, F = p.shape[0], faces.shape[0]
    x = (p[None] * (1 + 0.05 * torch.randn(B, V, 1, generator=g, device=dev))).contiguous()
    n = lighting.vertex_normals(x, faces).detach()
    leaves = [t.clone().requires_grad_(True) for t in (x, uv, n)]
    grad_out = torch.randn(B, V, 4, generator=g, device=dev)
    op = lambda a, b, c: lighting.vertex_tangents(a, b, faces, c)
    ref = lambda a, b, c: lighting._vertex_tangents(a, b, faces, c)

    def fwd(fn):
        with torch.no_grad():
            return fn(x, uv, n)

    def fwd_bwd(fn):
        for t in leaves:
            t.grad = None
        fn(*leaves).backward(grad_out)

    P = lambda t: ctypes.c_void_p(t.data_ptr())
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    ws_bytes = int(L.dirt_tangents_workspace_bytes(B, V, F))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    out = torch.empty(B * V, 4, device=dev)
    gv, gu, gn = torch.empty(B * V, 3, device=dev), torch.empty(B * V, 2, device=dev), torch.empty(B * V, 3, device=dev)
    tin = lambda: [P(x), 3, P(uv), 2, 0, P(n), 3, P(faces)]
    k_fwd = timed(lambda: L.dirt_tangents_forward(*tin(), P(out), P(ws), ws_bytes, B, V, F, stream()), args.steps)
    k_fwd_launches = L.dirt_last_launch_count()
    k_bwd = timed(lambda: L.dirt_tangents_backward(*tin(), P(grad_out), P(gv), P(gu), P(gn), P(ws), ws_bytes, B, V, F,
                                                   stream()), args.steps)
    k_bwd_launches = L.dirt_last_launch_count()
    op_fwd, torch_fwd = compare(lambda: fwd(op), lambda: fwd(ref), args.steps, args.rounds)
    op_fb, torch_fb = compare(lambda: fwd_bwd(op), lambda: fwd_bwd(ref), args.steps, args.rounds)
    fb, bb = tangent_bytes(B, V, F)
    return {'case': label, 'B': B, 'V': V, 'F': F, 'op_fwd_ms': op_fwd, 'torch_fwd_ms': torch_fwd,
            'op_fwd_bwd_ms': op_fb, 'torch_fwd_bwd_ms': torch_fb, 'kernel_fwd_ms': k_fwd, 'kernel_bwd_ms': k_bwd,
            'kernel_fwd_launches': k_fwd_launches, 'kernel_bwd_launches': k_bwd_launches,
            'op_launches': profile_launches(lambda: fwd_bwd(op)), 'torch_launches': profile_launches(lambda: fwd_bwd(ref)),
            'fwd_bytes': fb, 'bwd_bytes': bb,
            'kernel_fwd_of_peak': fb / (k_fwd * 1e-3) / 1e12 / PEAK_TBS,
            'kernel_bwd_of_peak': bb / (k_bwd * 1e-3) / 1e12 / PEAK_TBS,
            'op_held_mb': held_mb(lambda: op(*leaves)), 'torch_held_mb': held_mb(lambda: ref(*leaves)),
            'speedup_fwd': torch_fwd / op_fwd, 'speedup_fwd_bwd': torch_fb / op_fb}


def perturb_case(label, views, B, H, W, args, L, lighting, dev):
    g = torch.Generator(device=dev).manual_seed(1)
    N = B * H * W
    if views:
        gbuffer = torch.randn(B, H * W, 14, generator=g, device=dev)
        n, t, m = gbuffer[..., 3:6], gbuffer[..., 6:10], gbuffer[..., 10:13]
        base = [gbuffer]
    else:
        n, t, m = (torch.randn(B, H * W, k, generator=g, device=dev) for k in (3, 4, 3))
        base = [n, t, m]
    leaves = [b.clone().requires_grad_(True) for b in base]
    pick = (lambda l: (l[0][..., 3:6], l[0][..., 6:10], l[0][..., 10:13])) if views else (lambda l: tuple(l))
    grad_out = torch.randn(B, H * W, 3, generator=g, device=dev)
    op, ref = lighting.perturb_normals, lighting._perturb_normals

    def fwd(fn):
        with torch.no_grad():
            return fn(n, t, m)

    def fwd_bwd(fn):
        for l in leaves:
            l.grad = None
        fn(*pick(leaves)).backward(grad_out)

    P = lambda x: ctypes.c_void_p(x.data_ptr())
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    rows = [lighting._rows(a, k) for a, k in ((n, 3), (t, 4), (m, 3))]
    assert all(r.data_ptr() == a.data_ptr() for r, a in zip(rows, (n, t, m)))
    mi = lambda: [P(rows[0]), rows[0].stride(0), P(rows[1]), rows[1].stride(0), P(rows[2]), rows[2].stride(0)]
    out = torch.empty(N, 3, device=dev)
    gn, gt, gm = (torch.empty(N, k, device=dev) for k in (3, 4, 3))
    k_fwd = timed(lambda: L.dirt_normal_map_forward(*mi(), P(out), B, H * W, stream()), args.steps)
    k_fwd_launches = L.dirt_last_launch_count()
    k_bwd = timed(lambda: L.dirt_normal_map_backward(*mi(), P(grad_out), P(gn), P(gt), P(gm), B, H * W, stream()),
                  args.steps)
    k_bwd_launches = L.dirt_last_launch_count()
    op_fwd, torch_fwd = compare(lambda: fwd(op), lambda: fwd(ref), args.steps, args.rounds)
    op_fb, torch_fb = compare(lambda: fwd_bwd(op), lambda: fwd_bwd(ref), args.steps, args.rounds)
    fb, bb = perturb_bytes(N)
    return {'case': label, 'B': B, 'points': H * W, 'op_fwd_ms': op_fwd, 'torch_fwd_ms': torch_fwd,
            'op_fwd_bwd_ms': op_fb, 'torch_fwd_bwd_ms': torch_fb, 'kernel_fwd_ms': k_fwd, 'kernel_bwd_ms': k_bwd,
            'kernel_fwd_launches': k_fwd_launches, 'kernel_bwd_launches': k_bwd_launches,
            'op_launches': profile_launches(lambda: fwd_bwd(op)), 'torch_launches': profile_launches(lambda: fwd_bwd(ref)),
            'fwd_bytes': fb, 'bwd_bytes': bb,
            'kernel_fwd_of_peak': fb / (k_fwd * 1e-3) / 1e12 / PEAK_TBS,
            'kernel_bwd_of_peak': bb / (k_bwd * 1e-3) / 1e12 / PEAK_TBS,
            'op_held_mb': held_mb(lambda: op(*pick(leaves))), 'torch_held_mb': held_mb(lambda: ref(*pick(leaves))),
            'speedup_fwd': torch_fwd / op_fwd, 'speedup_fwd_bwd': torch_fb / op_fb}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('normalmapbench.py needs a CUDA device')
    from dirt_b200 import _lib, lighting
    L = _lib.lib()
    dev = torch.device('cuda', 0)
    name, limit = card()
    result = {'device': name, 'power_limit': limit, 'steps': args.steps, 'rounds': args.rounds, 'cases': []}
    cases = [lambda: tangent_case('a: tangents, seamed uv sphere 224 x 112, B=64, shared uvs', 224, 112, 64, args, L,
                                  lighting, dev),
             lambda: tangent_case('b: tangents, seamed uv sphere 1024 x 512, B=1', 1024, 512, 1, args, L, lighting, dev),
             lambda: perturb_case('c: perturb_normals, 64 x 512^2 points, contiguous', False, 64, 512, 512, args, L,
                                  lighting, dev),
             lambda: perturb_case('d: perturb_normals, 64 x 512^2 points, views of a 14-channel G-buffer', True, 64, 512,
                                  512, args, L, lighting, dev)]
    for case in cases:
        c = case()
        result['cases'].append(c)
        print(json.dumps(c), flush=True)
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
