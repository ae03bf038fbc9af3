"""Times the edge terms' CUDA path (edge lengths, normal consistency) against their torch restatements
(dirt_b200/mesh.py), and optionally sweeps the normal-consistency weight of examples/silhouette.py.

    python profiles/edgetermsbench.py [--steps 50] [--rounds 5] [--sweep MU,MU,...] [--runs 2] [--out FILE]

Workloads (laplacianbench.py's a-c):
  a  cfg3's icosphere-4 (V = 2562, F = 5120), B = 64 posed items as cfg3 lays them out: [64, V, 4]
  b  cfg5's displaced uv-sphere (V = 24866, F = 49728), B = 64 posed items [64, V, 3]
  c  uv_sphere(1024, 512) (V = 523266), B = 1: two rows of valence 1024
For each workload and op, alternating op and restatement in --rounds rounds of --steps calls each (the figures are
medians over the rounds):
  op_fwd_ms / op_fwd_bwd_ms        the public function through autograd (Python layer and allocations included)
  torch_fwd_ms / torch_fwd_bwd_ms  the same call with the restatement in its place
  kernel_fwd_ms / kernel_bwd_ms    the C ABI alone on preallocated buffers; the forward includes the adjacency build
  kernel_adjacency_ms              the adjacency build's kernels alone (torch.profiler, in a run of its own)
  op_launches / torch_launches     kernels and memsets per forward + backward (torch.profiler)
  *_bytes, *_of_peak               algorithmic bytes from shapes / kernel time, against the H100 SXM data sheet's 3.35 TB/s
  op_held_mb / torch_held_mb       device memory autograd holds between forward and backward (output included)
With --sweep, examples/silhouette.py's fit at lambda = 10 and each mu, --runs times each, plus (10, 0) and (0, 0): held-out
IoU, mean normal consistency and faces flipped.  CUDA events on the launching stream.  One JSON object with the card's
name and power limit.
"""
import argparse
import ctypes
import importlib.util
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lightbench import PEAK_TBS, card, compare, held_mb, timed   # noqa: E402

from laplacianbench import workloads   # noqa: E402
from normalsbench import profile   # noqa: E402


def algorithmic_bytes(B, V, F, consistency):
    """fwd: read the faces and each vertex's position once, write the per-edge values.  bwd: read the faces, the
    positions and grad_out, write the vertex gradients; the consistency backward also writes and reads its per-face
    dL/dn."""
    fwd = 12 * F + 12 * B * V + 12 * B * F
    bwd = 12 * F + 12 * B * V + 12 * B * F + 12 * B * V + (2 * 12 * B * F if consistency else 0)
    return fwd, bwd


def sweep(mus, runs, steps, dev):
    spec = importlib.util.spec_from_file_location('silhouette_example', os.path.join(ROOT, 'examples', 'silhouette.py'))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    out = []
    for run in range(runs):
        for weight, mu in [(10., 0.), (0., 0.)] + [(10., m) for m in mus]:
            r = ex.fit(weight, steps, device=dev, verbose=False, consistency=mu)
            r['run'] = run
            out.append(r)
            print(json.dumps(r), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--sweep', default=None, help='comma-separated normal-consistency weights for the example')
    ap.add_argument('--runs', type=int, default=2)
    ap.add_argument('--fit-steps', type=int, default=300)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('edgetermsbench.py needs a CUDA device')
    from dirt_b200 import _lib, mesh
    L = _lib.lib()
    dev = torch.device('cuda', 0)
    name, limit = card()
    result = {'device': name, 'power_limit': limit, 'steps': args.steps, 'rounds': args.rounds, 'cases': []}
    g = torch.Generator(device=dev).manual_seed(0)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for (label, vertices, faces), op_name in [(w, m) for w in workloads(dev) for m in mesh.EDGE_MODES]:
        op_fn, ref_fn = getattr(mesh, op_name), getattr(mesh, '_' + op_name)
        mode = mesh.EDGE_MODES[op_name]
        lead, V, F = vertices.shape[:-2], vertices.shape[-2], faces.shape[0]
        B = int(np.prod(lead)) if lead else 1
        leaf = vertices.clone().requires_grad_(True)
        grad_out = torch.randn(lead + (F, 3), generator=g, device=dev)

        def fwd(fn):
            with torch.no_grad():
                return fn(vertices, faces)

        def fwd_bwd(fn):
            leaf.grad = None
            fn(leaf, faces).backward(grad_out)

        # the ABI on preallocated buffers
        rows = vertices.view(-1, vertices.shape[-1])
        stride = rows.stride(0)
        out = torch.empty(B * F, 3, device=dev)
        grad = torch.empty(B * V, 3, device=dev)
        ws_bytes = int(L.dirt_edge_terms_workspace_bytes(B, V, F))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        k_fwd_call = lambda: L.dirt_edge_terms_forward(mode, p(rows), stride, p(faces), p(out), p(ws), ws_bytes, B, V,
                                                       F, stream())
        k_bwd_call = lambda: L.dirt_edge_terms_backward(mode, p(rows), stride, p(faces), p(grad_out), p(grad), p(ws),
                                                        ws_bytes, B, V, F, stream())
        k_fwd = timed(k_fwd_call, args.steps)
        k_fwd_launches = L.dirt_last_launch_count()
        k_bwd = timed(k_bwd_call, args.steps)
        k_bwd_launches = L.dirt_last_launch_count()
        op_fwd, torch_fwd = compare(lambda: fwd(op_fn), lambda: fwd(ref_fn), args.steps, args.rounds)
        op_fb, torch_fb = compare(lambda: fwd_bwd(op_fn), lambda: fwd_bwd(ref_fn), args.steps, args.rounds)
        op_launches, adjacency = profile(lambda: fwd_bwd(op_fn), 10)
        torch_launches, _ = profile(lambda: fwd_bwd(ref_fn), 10)
        fb, bb = algorithmic_bytes(B, V, F, mode == _lib.NORMAL_CONSISTENCY)
        case = {'case': label, 'op': op_name, 'B': B, 'V': V, 'F': F, 'op_fwd_ms': op_fwd,
                'torch_fwd_ms': torch_fwd, 'op_fwd_bwd_ms': op_fb, 'torch_fwd_bwd_ms': torch_fb, 'kernel_fwd_ms': k_fwd,
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
    if args.sweep:
        result['example'] = {'fit_steps': args.fit_steps,
                             'fits': sweep([float(m) for m in args.sweep.split(',')], args.runs, args.fit_steps, dev)}
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            f.write(json.dumps(result, indent=1) + '\n')


if __name__ == '__main__':
    main()
