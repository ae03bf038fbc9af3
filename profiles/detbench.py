"""Cost of the deterministic backward pass (DESIGN.md §7.4): the default and the deterministic RasteriseGrad call,
alternated in one run on the benched workloads, the public API's forward + backward with torch's deterministic
algorithms on, and peak memory.  Writes one JSON document (with the card's name and power limit) to stdout or --out.

    python profiles/detbench.py [--iters 20] [--out profiles/h100_deterministic.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

WORKLOADS = {
    'cfg3': ('config3', dict(batch=64, width=512, height=512, background='uniform')),
    'cfg4': ('config4', dict(batch=32, width=512, height=512)),
    'cfg5': ('config5', dict(batch=64, width=1024, height=1024)),
    'cube': ('cube_batch', dict(batch=64, width=640, height=480)),
}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn, iters):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / iters


def run(name, iters):
    from dirt_b200 import scenes
    from dirt_b200 import rasterise_ops as ops
    import dirt_b200 as dirt
    builder, kw = WORKLOADS[name]
    s = getattr(scenes, builder)(**kw)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in s.items()}
    pixels, ids, ws = ops.rasterise_forward_raw(t['background'], t['vertices'], t['vertex_colors'], t['faces'],
                                                return_workspace=True)
    gp = torch.randn_like(pixels)
    groups = ops.default_channel_groups(int(pixels.shape[3]))

    def bwd(det):
        return lambda: ops.rasterise_backward_raw(t['vertices'], t['faces'], pixels, gp, ids, groups, ws, deterministic=det)

    for det in (False, True):
        bwd(det)()
    torch.cuda.synchronize()
    rounds = {'default': [], 'deterministic': []}
    for _ in range(5):   # alternated
        rounds['default'].append(timed(bwd(False), iters))
        rounds['deterministic'].append(timed(bwd(True), iters))
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    bwd(True)()
    torch.cuda.synchronize()
    peak_det = torch.cuda.max_memory_allocated() - base
    torch.cuda.reset_peak_memory_stats()
    bwd(False)()
    torch.cuda.synchronize()
    peak_def = torch.cuda.max_memory_allocated() - base

    # kernel times of one deterministic call
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            bwd(True)()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA or 'kernel' in e.key or 'Memset' in e.key:
            us = getattr(e, 'device_time_total', getattr(e, 'cuda_time_total', 0.0))
            kernels[e.key[:90]] = round(us / 3 / 1000.0, 4)

    def api(flag):
        torch.use_deterministic_algorithms(flag)
        try:
            bg = t['background'].clone().requires_grad_(True)
            v = t['vertices'].clone().requires_grad_(True)
            c = t['vertex_colors'].clone().requires_grad_(True)
            out = dirt.rasterise_batch(bg, v, c, t['faces'])
            out.backward(gp)
        finally:
            torch.use_deterministic_algorithms(False)

    api(True)
    api(False)
    api_rounds = {'default': [], 'deterministic_flag_on': []}
    for _ in range(3):
        api_rounds['default'].append(timed(lambda: api(False), max(2, iters // 4)))
        api_rounds['deterministic_flag_on'].append(timed(lambda: api(True), max(2, iters // 4)))
    med = {k: float(np.median(v)) for k, v in rounds.items()}
    amed = {k: float(np.median(v)) for k, v in api_rounds.items()}
    return {
        'backward_ms': rounds, 'backward_ms_median': med, 'ratio': med['deterministic'] / med['default'],
        'public_api_fwd_bwd_ms': api_rounds, 'public_api_fwd_bwd_ms_median': amed,
        'public_api_ratio': amed['deterministic_flag_on'] / amed['default'],
        'peak_extra_bytes': {'default': int(peak_def), 'deterministic': int(peak_det)},
        'scratch_bytes': int(ops._lib.lib().dirt_rasterise_backward_deterministic_bytes(
            *pixels.shape, t['vertices'].shape[1], t['faces'].shape[1])),
        'kernels_ms_per_call': kernels,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--workloads', default='cfg3,cfg4,cfg5,cube')
    ap.add_argument('--out')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'detbench needs a CUDA device'
    doc = {'card': card(), 'workloads': {}}
    for name in args.workloads.split(','):
        doc['workloads'][name] = run(name, args.iters)
        print(name, json.dumps({k: doc['workloads'][name][k] for k in ('backward_ms_median', 'ratio', 'public_api_ratio')}),
              flush=True)
    text = json.dumps(doc, indent=1)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(text + '\n')
    else:
        print(text)


if __name__ == '__main__':
    main()
