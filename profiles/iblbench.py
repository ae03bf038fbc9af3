"""Times split-sum GGX image-based lighting (DESIGN.md §7.12): the prefilter, and the 'ggx' lookup against 'trilinear'.

    python profiles/iblbench.py [--steps 5] [--rounds 3] [--out FILE]

  prefilter_ms        dirt_cubemap_ggx_prefilter of one shared 6 x S^2 map, C = 3, S = 256 and 1024 (box pyramid, texel
                      table, levels 1 .. L-1 and W), with the texel pairs and FP32 operations counted from the shapes
                      by `pairs` below, and the achieved rate against the H100 SXM data sheet's 67 TFLOP/s
  op_fwd_ms / op_fwd_bwd_ms   sample_cubemap(..., 'ggx', roughness=...) through autograd, N = 64 x 512^2 reflection
                      lookups (profiles/cubebench.py's) into the S = 256 map, roughness uniform in [0, 1], gradients to
                      the cube map, directions and roughness; trilinear_* the same with mode 'trilinear' at
                      lod = roughness * (L-1); det_fwd_bwd_ms under torch.use_deterministic_algorithms(True)
  op_held_mb          device memory autograd holds between forward and backward (output included)
CUDA events on the launching stream, medians of alternating rounds.  One JSON object with the card's name and power
limit.
"""
import argparse
import ctypes
import json
import math
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))
from cubebench import directions  # noqa: E402
from lightbench import card, compare, held_mb, timed  # noqa: E402

PEAK_FP32_TFLOPS = 67.0
# per pair: the cosine (1 mul + 2 fma), the support test, k (1 sub + 1 fma), k^2, c * Omega, 1 division, W, C fma
FLOPS_PER_PAIR = lambda C: 5 + 3 + 1 + 1 + 1 + 1 + 2 * C


def levels(S):
    L = 1
    while S >> (L - 1) > 0 and (S >> (L - 1)) % 2 == 0:
        L += 1
    return L


def pairs(S):
    """Texel pairs summed by the prefilter of a 6 x S^2 map, estimated from the lobes' support cones: each output
    texel of level k sees 2 pi (1 - c_k) / (4 pi) of the 6 S_s^2 source texels."""
    L = levels(S)
    ss = max([k for k in range(L) if (S >> k) >= 16] or [0])
    total = 0.
    for k in range(1, L):
        a = max(k / (L - 1), 0.045)
        a2 = a ** 4
        ck = 0. if a2 >= 1 else max(0., 1 - 2 * (math.sqrt(1000) - 1) * a2 / (1 - a2))
        s = min(k, ss)
        total += 6 * (S >> k) ** 2 * 6 * (S >> s) ** 2 * (1 - ck) / 2
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import dirt_b200 as dirt
    from dirt_b200 import _lib
    L_ = _lib.lib()
    dev = torch.device('cuda', 0)
    name, limit = card()
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    result = {'card': name, 'power_limit': limit, 'prefilter': []}
    gen = torch.Generator(device=dev).manual_seed(0)
    for S in (256, 1024):
        C = 3
        cube = torch.rand(1, 6, S, S, C, generator=gen, device=dev)
        atlas = torch.empty(int(L_.dirt_cubemap_ggx_atlas_bytes(1, S, C)) // 4, device=dev)
        run = lambda: L_.dirt_cubemap_ggx_prefilter(ctypes.c_void_p(cube.data_ptr()), ctypes.c_void_p(atlas.data_ptr()),
                                                    1, S, C, stream())
        assert run() == 0
        ms = statistics.median(timed(run, args.steps) for _ in range(args.rounds))
        n = pairs(S)
        flops = n * FLOPS_PER_PAIR(C)
        result['prefilter'].append({'S': S, 'C': C, 'prefilter_ms': ms, 'pairs_estimate': n, 'flops_estimate': flops,
                                    'tflops': flops / ms / 1e9, 'of_fp32_peak': flops / ms / 1e9 / PEAK_FP32_TFLOPS,
                                    'bound': 'FP32 arithmetic (%.3g bytes of maps against %.3g FLOPs)'
                                             % (4 * 6 * S * S * C * 8 / 3, flops)})
        print(json.dumps(result['prefilter'][-1]), flush=True)
        del atlas
    S, C = 256, 3
    lv = levels(S)
    cube = torch.rand(6, S, S, C, generator=gen, device=dev)
    d = directions('reflection', 64, 512, 512, dev, gen).reshape(-1, 3).contiguous()
    rough = torch.rand(d.shape[0], generator=gen, device=dev)
    g = torch.randn(d.shape[0], C, generator=gen, device=dev)

    def fwd(mode):
        if mode == 'ggx':
            return lambda: dirt.sample_cubemap(cube, d, 'ggx', roughness=rough)
        return lambda: dirt.sample_cubemap(cube, d, 'trilinear', lod=rough * float(lv - 1))

    def fwd_bwd(mode):
        def run():
            c, x, r = (t.detach().requires_grad_(True) for t in (cube, d, rough))
            out = (dirt.sample_cubemap(c, x, 'ggx', roughness=r) if mode == 'ggx' else
                   dirt.sample_cubemap(c, x, 'trilinear', lod=r * float(lv - 1)))
            out.backward(g)
        return run

    op_f, tri_f = compare(fwd('ggx'), fwd('trilinear'), args.steps, args.rounds)
    op_fb, tri_fb = compare(fwd_bwd('ggx'), fwd_bwd('trilinear'), args.steps, args.rounds)
    torch.use_deterministic_algorithms(True)
    try:
        det_fb = statistics.median(timed(fwd_bwd('ggx'), args.steps) for _ in range(args.rounds))
    finally:
        torch.use_deterministic_algorithms(False)

    def held():
        c, x, r = (t.detach().requires_grad_(True) for t in (cube, d, rough))
        return dirt.sample_cubemap(c, x, 'ggx', roughness=r)

    result['lookup'] = {'S': S, 'C': C, 'N': d.shape[0], 'op_fwd_ms': op_f, 'trilinear_fwd_ms': tri_f,
                        'op_fwd_bwd_ms': op_fb, 'trilinear_fwd_bwd_ms': tri_fb, 'det_fwd_bwd_ms': det_fb,
                        'op_held_mb': held_mb(held)}
    print(json.dumps(result['lookup']), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)
            f.write('\n')


if __name__ == '__main__':
    main()
