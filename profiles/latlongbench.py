"""Times the lat-long to cube-map conversion (DESIGN.md §7.13), its kernels and the torch restatement.

    python profiles/latlongbench.py [--steps 10] [--rounds 3] [--out FILE]

Per case (C = 3: 1024 x 2048 -> 512 and 2048 x 4096 -> 1024 shared, and 8 per-item panoramas of 1024 x 2048 -> 512):
  fwd_kernel_ms / bwd_kernel_ms   dirt_latlong_to_cubemap / _backward called directly, CUDA events around `steps`
                      calls; *_roofline is the least time the algorithmic bytes (`bytes_fwd`: the panorama read once,
                      the cube map written once; the backward the reverse) take at the H100 SXM's 3.35 TB/s, over the
                      kernel time
  op_fwd_ms / op_fwd_bwd_ms and ref_fwd_ms / ref_fwd_bwd_ms   latlong_to_cubemap through autograd against
                      tests/latlong_restatement.py in float32 on the GPU (the gradient to the panorama), medians of
                      alternating rounds
  op_held_mb / ref_held_mb        device memory autograd holds between forward and backward (output included)
The forward's bits are checked against the restatement's at every size.  One JSON object with the card's name and
power limit.
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
from lightbench import card, compare, held_mb, timed  # noqa: E402

HBM_TBPS = 3.35
CASES = [(1024, 2048, 512, None), (2048, 4096, 1024, None), (1024, 2048, 512, 8)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('latlongbench needs a CUDA device')
    import latlong_restatement as ll
    import dirt_b200 as dirt
    from dirt_b200 import _lib, build
    build.build()
    L = _lib.lib()
    dev = torch.device('cuda', 0)
    name, limit = card()
    result = {'card': name, 'power_limit': limit, 'steps': args.steps, 'rounds': args.rounds, 'cases': []}
    C = 3
    for H, W, S, batch in CASES:
        TB = batch or 1
        g = torch.Generator(device=dev).manual_seed(H + S)
        pan = torch.rand((TB, H, W, C), generator=g, device=dev)
        grad = torch.randn((TB, 6, S, S, C), generator=g, device=dev)
        cube = torch.empty_like(grad)
        gp = torch.empty_like(pan)
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        fwd = lambda: _lib.check(L.dirt_latlong_to_cubemap(p(pan), p(cube), TB, H, W, S, C, stream), 'fwd')
        bwd = lambda: _lib.check(L.dirt_latlong_to_cubemap_backward(p(grad), p(gp), TB, H, W, S, C, stream), 'bwd')
        fwd_ms, bwd_ms = timed(fwd, args.steps), timed(bwd, args.steps)
        bytes_fwd = 4 * TB * (H * W + 6 * S * S) * C
        x = pan if batch else pan[0]
        assert torch.equal(dirt.latlong_to_cubemap(x, S).view(torch.int32), ll.to_cubemap(x, S).view(torch.int32))
        gx = grad if batch else grad[0]

        def op_fwd():
            return dirt.latlong_to_cubemap(x, S)

        def ref_fwd():
            return ll.to_cubemap(x, S)

        def fwd_bwd(f):
            def run():
                q = x.detach().requires_grad_(True)
                torch.autograd.grad((f(q, S) * gx).sum(), q)
            return run

        op_f, ref_f = compare(op_fwd, ref_fwd, args.steps, args.rounds)
        op_fb, ref_fb = compare(fwd_bwd(dirt.latlong_to_cubemap), fwd_bwd(ll.to_cubemap), max(1, args.steps // 2),
                                args.rounds)
        xq = x.detach().requires_grad_(True)
        case = {'H': H, 'W': W, 'S': S, 'C': C, 'items': batch, 'n': ll.samples(H, W, S),
                'fwd_kernel_ms': fwd_ms, 'bwd_kernel_ms': bwd_ms, 'bytes_fwd': bytes_fwd,
                'fwd_roofline': bytes_fwd / (HBM_TBPS * 1e12) / (fwd_ms * 1e-3),
                'bwd_roofline': bytes_fwd / (HBM_TBPS * 1e12) / (bwd_ms * 1e-3),
                'op_fwd_ms': op_f, 'ref_fwd_ms': ref_f, 'op_fwd_bwd_ms': op_fb, 'ref_fwd_bwd_ms': ref_fb,
                'op_held_mb': held_mb(lambda: dirt.latlong_to_cubemap(xq, S)),
                'ref_held_mb': held_mb(lambda: ll.to_cubemap(xq, S))}
        result['cases'].append(case)
        print(json.dumps(case), flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(json.dumps(result, indent=1) + '\n')


if __name__ == '__main__':
    main()
