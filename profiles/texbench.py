"""Times dirt_b200.sample_texture against the torch restatement of examples/textured.py.

    python profiles/texbench.py [--steps 20] [--out FILE]

Workload: N = 64 x 512^2 lookups (one per pixel of a cfg3-sized G-buffer), C = 3, one shared texture of 1024^2 and of
256^2 texels, and two index patterns: `gbuffer` (each image shows a rotated, scaled patch of the texture, about one texel
per pixel: neighbouring pixels read neighbouring texels) and `random` (uniform over the texture).  For each case:
  op_fwd_ms / op_fwd_bwd_ms      dirt_b200.sample_texture through autograd (allocations and the Python layer included)
  torch_fwd_ms / torch_fwd_bwd_ms the restatement, same calls
  kernel_fwd_ms / kernel_bwd_ms   the C ABI alone on preallocated buffers (backward: both gradients, memset included)
  *_tbs                           algorithmic bytes / kernel time, against the H100 SXM data sheet's 3.35 TB/s
CUDA events on the launching stream, averaged over --steps calls after warm-up.  One JSON object with the card's name and
power limit.
"""
import argparse
import ctypes
import importlib.util
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK_TBS = 3.35   # H100 SXM data sheet HBM3 bandwidth


def algorithmic_bytes(N, texels, C):
    """fwd: read the index pair, write C floats per lookup, read the texture once.
    bwd: read the index pair and C floats of grad_out, write the index gradient per lookup; read the texture once (index
    gradient), zero and write grad_texture once."""
    fwd = N * (8 + 4 * C) + texels * 4 * C
    bwd = N * (8 + 4 * C + 8) + 3 * texels * 4 * C
    return fwd, bwd


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = 'unknown'
    return name, limit


def timed(fn, steps, warmup=3):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def gbuffer_indices(B, H, W, size, device, seed=0):
    g = torch.Generator(device=device).manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(H, device=device, dtype=torch.float32),
                            torch.arange(W, device=device, dtype=torch.float32), indexing='ij')
    angle = torch.rand(B, 1, 1, generator=g, device=device) * 6.283
    scale = (0.8 + 0.4 * torch.rand(B, 1, 1, generator=g, device=device)) * size / max(H, W)
    origin = torch.rand(B, 1, 2, generator=g, device=device) * size
    r = (torch.cos(angle) * ys - torch.sin(angle) * xs) * scale
    c = (torch.sin(angle) * ys + torch.cos(angle) * xs) * scale
    return (torch.stack([r, c], -1).reshape(B, -1, 2) + origin).reshape(-1, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import dirt_b200 as dirt
    from dirt_b200 import _lib
    spec = importlib.util.spec_from_file_location('textured_example', os.path.join(ROOT, 'examples', 'textured.py'))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    L = _lib.lib()
    dev = torch.device('cuda', 0)
    B, H, W, C = 64, 512, 512, 3
    N = B * H * W
    name, limit = card()
    result = {'device': name, 'power_limit': limit, 'lookups': N, 'channels': C, 'steps': args.steps, 'cases': []}
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    for size in (1024, 256):
        texture = torch.rand(size, size, C, device=dev)
        for pattern in ('gbuffer', 'random'):
            if pattern == 'gbuffer':
                indices = gbuffer_indices(B, H, W, size, dev)
            else:
                indices = torch.rand(N, 2, device=dev) * size
            grad_out = torch.randn(N, C, device=dev)
            out = torch.empty(N, C, device=dev)
            grad_texture = torch.empty_like(texture)
            grad_indices = torch.empty_like(indices)
            stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            k_fwd = timed(lambda: L.dirt_texture_sample(p(texture), p(indices), p(out), 1, size, size, C, 1, N, 0, stream()),
                          args.steps)
            k_bwd = timed(lambda: L.dirt_texture_sample_backward(p(texture), p(indices), p(grad_out), p(grad_texture),
                                                                 p(grad_indices), 1, size, size, C, 1, N, 0, stream()),
                          args.steps)
            tex_p, idx_p = texture.clone().requires_grad_(True), indices.clone().requires_grad_(True)

            def fwd(fn):
                with torch.no_grad():
                    fn(texture, indices)

            def fwd_bwd(fn):
                tex_p.grad, idx_p.grad = None, None
                fn(tex_p, idx_p).backward(grad_out)

            fb, bb = algorithmic_bytes(N, size * size, C)
            case = {'texture': size, 'pattern': pattern,
                    'op_fwd_ms': timed(lambda: fwd(dirt.sample_texture), args.steps),
                    'op_fwd_bwd_ms': timed(lambda: fwd_bwd(dirt.sample_texture), args.steps),
                    'torch_fwd_ms': timed(lambda: fwd(ex.sample_texture), args.steps),
                    'torch_fwd_bwd_ms': timed(lambda: fwd_bwd(ex.sample_texture), args.steps),
                    'kernel_fwd_ms': k_fwd, 'kernel_bwd_ms': k_bwd,
                    'fwd_bytes': fb, 'bwd_bytes': bb}
            case['kernel_fwd_tbs'] = fb / (k_fwd * 1e-3) / 1e12
            case['kernel_bwd_tbs'] = bb / (k_bwd * 1e-3) / 1e12
            case['kernel_fwd_of_peak'] = case['kernel_fwd_tbs'] / PEAK_TBS
            case['kernel_bwd_of_peak'] = case['kernel_bwd_tbs'] / PEAK_TBS
            case['speedup_fwd'] = case['torch_fwd_ms'] / case['op_fwd_ms']
            case['speedup_fwd_bwd'] = case['torch_fwd_bwd_ms'] / case['op_fwd_bwd_ms']
            result['cases'].append(case)
            print(json.dumps(case), flush=True)
            del tex_p, idx_p
            torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(json.dumps(result, indent=1) + '\n')


if __name__ == '__main__':
    main()
