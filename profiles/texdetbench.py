"""Cost of the deterministic texture backward pass (DESIGN.md §7.5): the default and the deterministic
dirt_texture_sample_backward call, alternated in one run, on texbench's four cases (64 x 512^2 lookups, C = 3, one
1024^2 or 256^2 texture, gbuffer or random indices), a 16^2 texture over 64 x 512^2 pixels, the worst case (every lookup
on one texel), and per-item 64 x 256^2 textures; the public API's forward + backward with torch's deterministic
algorithms on and off; the scratch bytes; and, in a separate profiled call, the kernel time per phase.  Writes one JSON
document (with the card's name and power limit, read in the same run) to stdout or --out.

    python profiles/texdetbench.py [--iters 10] [--rounds 3] [--out profiles/h100_texture_deterministic.json]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))

import torch  # noqa: E402

from texbench import card, gbuffer_indices  # noqa: E402

B, H, W, C = 64, 512, 512, 3


def timed(fn, iters):
    fn()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / iters


def cases(dev):
    """name -> (texture [TB, TH, TW, C], indices [B, N, 2])"""
    g = torch.Generator(device=dev).manual_seed(0)
    n = B * H * W
    for size in (1024, 256):
        tex = torch.rand(1, size, size, C, generator=g, device=dev)
        yield '%d^2 gbuffer' % size, tex, gbuffer_indices(B, H, W, size, dev).reshape(B, -1, 2)
        yield '%d^2 random' % size, tex, (torch.rand(n, 2, generator=g, device=dev) * size).reshape(B, -1, 2)
    ys, xs = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing='ij')
    one = torch.stack([(ys + 0.5) / H * 16, (xs + 0.5) / W * 16], -1).reshape(1, -1, 2).expand(B, -1, -1)
    yield '16^2 over 512^2', torch.rand(1, 16, 16, C, generator=g, device=dev), one.contiguous()
    yield 'one texel', torch.rand(1, 1024, 1024, C, generator=g, device=dev), \
        torch.tensor([300.25, 700.5], device=dev).expand(B, H * W, 2).contiguous()
    yield 'per-item 64 x 256^2', torch.rand(B, 256, 256, C, generator=g, device=dev), \
        gbuffer_indices(B, H, W, 256, dev).reshape(B, -1, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import dirt_b200 as dirt
    from dirt_b200 import _lib
    L = _lib.lib()
    dev = torch.device('cuda', 0)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    result = {'device': card(), 'iters': args.iters, 'rounds': args.rounds, 'cases': []}
    for name, tex, idx in cases(dev):
        TB, TH, TW, _ = tex.shape
        N = idx.shape[1]
        gout = torch.randn(B, N, C, device=dev)
        gt, gi = torch.empty_like(tex), torch.empty_like(idx)
        nbytes = int(L.dirt_texture_sample_backward_deterministic_bytes(TB, TH, TW, C, B, N, 0))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)

        def default():
            assert L.dirt_texture_sample_backward(p(tex), p(idx), p(gout), p(gt), p(gi), TB, TH, TW, C, B, N, 0, stream()) == 0

        def det():
            assert L.dirt_texture_sample_backward_deterministic(p(tex), p(idx), p(gout), p(gt), p(gi), TB, TH, TW, C, B, N,
                                                                0, p(scratch), nbytes, stream()) == 0

        rounds = {'default': [], 'deterministic': []}
        for _ in range(args.rounds):
            rounds['default'].append(timed(default, args.iters))
            rounds['deterministic'].append(timed(det, args.iters))
        med = {k: sorted(v)[len(v) // 2] for k, v in rounds.items()}
        # kernel time per phase of one deterministic call, profiled apart from the timings above
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            det()
            torch.cuda.synchronize()
        phases = {}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            key = next((k for k in ('tex_sort_hist', 'tex_sort_scan', 'tex_sort_scatter', 'tex_segment_bounds',
                                    'tex_det_gather', 'tex_det_chunk', 'tex_det_finish', 'texture_backward_kernel')
                        if k in e.name), 'other')
            phases[key] = phases.get(key, 0.0) + e.device_time / 1e3
        # the public API, forward + backward of both gradients, torch's flag on and off
        tex_p = (tex if TB > 1 else tex[0]).clone().requires_grad_(True)
        idx_p = (idx if TB > 1 else idx).clone().requires_grad_(True)

        def api():
            tex_p.grad, idx_p.grad = None, None
            dirt.sample_texture(tex_p, idx_p).backward(gout.reshape(idx_p.shape[:-1] + (C,)))

        api_rounds = {'flag_off': [], 'flag_on': []}
        for _ in range(args.rounds):
            for key, flag in (('flag_off', False), ('flag_on', True)):
                torch.use_deterministic_algorithms(flag)
                try:
                    api_rounds[key].append(timed(api, args.iters))
                finally:
                    torch.use_deterministic_algorithms(False)
        amed = {k: sorted(v)[len(v) // 2] for k, v in api_rounds.items()}
        case = {'case': name, 'textures': TB, 'texels': TH * TW, 'lookups': B * N, 'channels': C,
                'backward_ms': rounds, 'backward_ms_median': med, 'ratio': med['deterministic'] / med['default'],
                'phase_ms': phases, 'public_api_fwd_bwd_ms': api_rounds, 'public_api_fwd_bwd_ms_median': amed,
                'public_api_ratio': amed['flag_on'] / amed['flag_off'], 'scratch_bytes': nbytes}
        result['cases'].append(case)
        print(json.dumps({k: case[k] for k in ('case', 'backward_ms_median', 'ratio', 'public_api_ratio', 'phase_ms')}),
              flush=True)
        del scratch, tex_p, idx_p
        torch.cuda.empty_cache()
    print(json.dumps({'device': result['device']}))
    if args.out:
        with open(args.out, 'w') as f:
            f.write(json.dumps(result, indent=1) + '\n')


if __name__ == '__main__':
    main()
