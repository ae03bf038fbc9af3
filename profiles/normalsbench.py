"""Times the vertex normals' CUDA path against their torch restatement (dirt_b200/lighting.py).

    python profiles/normalsbench.py [--steps 50] [--rounds 5] [--out FILE]

Workloads:
  a  vertex_normals, cfg3's icosphere-4 (V = 2562, F = 5120), B = 64 posed items as cfg3 lays them out: [64, V, 4]
  b  vertex_normals, cfg5's displaced uv-sphere (V = 24866, F = 49728), B = 64 posed items [64, V, 3]
  c  vertex_normals, uv_sphere(1024, 512), B = 1: two rows of valence 1024
  d  vertex_normals_pre_split, the split icosphere-4, B = 64 ([64, 3F, 3])
For each, alternating op and restatement in --rounds rounds of --steps calls each (the figures are medians over the
rounds):
  op_fwd_ms / op_fwd_bwd_ms        the public function through autograd (Python layer and allocations included)
  torch_fwd_ms / torch_fwd_bwd_ms  the same call with the restatement in its place
  kernel_fwd_ms / kernel_bwd_ms    the C ABI alone on preallocated buffers; the forward includes the adjacency build
  kernel_adjacency_ms              the adjacency build's kernels alone (torch.profiler, in a run of its own)
  op_launches / torch_launches     kernels and memsets per forward + backward (torch.profiler)
  *_bytes, *_of_peak               algorithmic bytes from shapes / kernel time, against the H100 SXM data sheet's 3.35 TB/s
  op_held_mb / torch_held_mb       device memory autograd holds between forward and backward (output included)
CUDA events on the launching stream.  One JSON object with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lightbench import PEAK_TBS, card, compare, held_mb, timed   # noqa: E402

ADJACENCY_KERNELS = ('count_kernel', 'scan_kernel', 'fill_kernel', 'rank_kernel')


def algorithmic_bytes(B, V, F, pre_split):
    """fwd: read the faces and each vertex's position once, write the normals.  bwd: read the faces, the positions and
    grad_normals, write the vertex gradients; the average mode also writes and reads its per-vertex sum gradients."""
    fwd = 12 * F + 12 * B * V + 12 * B * V
    bwd = 12 * F + 3 * 12 * B * V + (0 if pre_split else 2 * 12 * B * V)
    return fwd, bwd


def workloads(dev):
    from dirt_b200 import scenes
    v4, f4 = scenes.icosphere(4)
    a, _ = scenes._posed_sphere_batch(v4, f4, 64, 512, 512, 1)
    v5, f5 = scenes.uv_sphere(224, 112, displacement=0.1)
    b, _ = scenes._posed_sphere_batch(v5, f5, 64, 1024, 1024, 3, ndc_radius=0.68)
    vc, fc = scenes.uv_sphere(1024, 512)
    split = a[:, f4.reshape(-1)][..., :3]
    t = lambda x: torch.tensor(np.ascontiguousarray(x), dtype=torch.float32, device=dev)
    faces = lambda f: torch.tensor(f, dtype=torch.int32, device=dev)
    return [('a: icosphere-4, B=64, [64, V, 4]', False, t(a), faces(f4)),
            ('b: cfg5 uv-sphere, B=64', False, t(b[..., :3]), faces(f5)),
            ('c: uv_sphere(1024, 512), B=1', False, t(vc), faces(fc)),
            ('d: pre-split, split icosphere-4, B=64', True,  t(split),
             faces(np.arange(3 * len(f4), dtype=np.int32).reshape(-1, 3)))]


def profile(fn, steps):
    """Per call of fn: the number of kernels and memsets, and the device time of the kernels whose names contain any of
    ADJACENCY_KERNELS."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    launches, adjacency_us = 0, 0.
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        launches += 1
        if any(k in e.name for k in ADJACENCY_KERNELS):
            adjacency_us += e.device_time
    return launches / steps, adjacency_us / steps / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('normalsbench.py needs a CUDA device')
    from dirt_b200 import _lib, lighting
    L = _lib.lib()
    dev = torch.device('cuda', 0)
    name, limit = card()
    result = {'device': name, 'power_limit': limit, 'steps': args.steps, 'rounds': args.rounds, 'cases': []}
    g = torch.Generator(device=dev).manual_seed(0)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for label, pre_split, vertices, faces in workloads(dev):
        op_fn = lighting.vertex_normals_pre_split if pre_split else lighting.vertex_normals
        ref_fn = lighting._vertex_normals_pre_split if pre_split else lighting._vertex_normals
        mode = _lib.NORMALS_PRE_SPLIT if pre_split else _lib.NORMALS_AVERAGE
        lead, V, F = vertices.shape[:-2], vertices.shape[-2], faces.shape[0]
        B = int(np.prod(lead)) if lead else 1
        leaf = vertices.clone().requires_grad_(True)
        grad_out = torch.randn(lead + (V, 3), generator=g, device=dev)

        def fwd(fn):
            with torch.no_grad():
                return fn(vertices, faces)

        def fwd_bwd(fn):
            leaf.grad = None
            fn(leaf, faces).backward(grad_out)

        # the ABI on preallocated buffers
        rows = vertices.view(-1, vertices.shape[-1])
        stride = rows.stride(0)
        out = torch.empty(B * V, 3, device=dev)
        grad = torch.empty(B * V, 3, device=dev)
        ws_bytes = int(L.dirt_normals_workspace_bytes(B, V, F))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        k_fwd_call = lambda: L.dirt_normals_forward(mode, p(rows), stride, p(faces), p(out), p(ws), ws_bytes, B, V, F,
                                                    stream())
        k_bwd_call = lambda: L.dirt_normals_backward(mode, p(rows), stride, p(faces), p(grad_out), p(grad), p(ws),
                                                     ws_bytes, B, V, F, stream())
        k_fwd = timed(k_fwd_call, args.steps)
        k_fwd_launches = L.dirt_last_launch_count()
        k_bwd = timed(k_bwd_call, args.steps)
        k_bwd_launches = L.dirt_last_launch_count()
        op_fwd, torch_fwd = compare(lambda: fwd(op_fn), lambda: fwd(ref_fn), args.steps, args.rounds)
        op_fb, torch_fb = compare(lambda: fwd_bwd(op_fn), lambda: fwd_bwd(ref_fn), args.steps, args.rounds)
        op_launches, adjacency = profile(lambda: fwd_bwd(op_fn), 10)
        torch_launches, _ = profile(lambda: fwd_bwd(ref_fn), 10)
        fb, bb = algorithmic_bytes(B, V, F, pre_split)
        case = {'case': label, 'B': B, 'V': V, 'F': F, 'op_fwd_ms': op_fwd, 'torch_fwd_ms': torch_fwd,
                'op_fwd_bwd_ms': op_fb, 'torch_fwd_bwd_ms': torch_fb, 'kernel_fwd_ms': k_fwd,
                'kernel_adjacency_ms': adjacency, 'kernel_bwd_ms': k_bwd,
                'kernel_fwd_launches': k_fwd_launches, 'kernel_bwd_launches': k_bwd_launches,
                'op_launches': op_launches, 'torch_launches': torch_launches, 'fwd_bytes': fb, 'bwd_bytes': bb,
                'kernel_fwd_of_peak': fb / (k_fwd * 1e-3) / 1e12 / PEAK_TBS,
                'kernel_bwd_of_peak': bb / (k_bwd * 1e-3) / 1e12 / PEAK_TBS,
                'op_held_mb': held_mb(lambda: op_fn(leaf, faces)),
                'torch_held_mb': held_mb(lambda: ref_fn(leaf, faces))}
        case['speedup_fwd'] = torch_fwd / op_fwd
        case['speedup_fwd_bwd'] = torch_fb / op_fb
        result['cases'].append(case)
        print(json.dumps(case), flush=True)
        del leaf, out, grad, ws
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            f.write(json.dumps(result, indent=1) + '\n')


if __name__ == '__main__':
    main()
