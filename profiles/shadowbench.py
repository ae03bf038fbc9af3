"""Times shadow_visibility (dirt_b200/lighting.py, DESIGN.md §7.15) against its torch restatement.

    python profiles/shadowbench.py [--steps 10] [--rounds 3] [--out FILE]

Workload: 64 x 512^2 points, each item a 512 x 512 grid over 90% of the light's view (light-clip x, y in [-0.9, 0.9],
z uniform), looked up in a 1024^2 map per item or in one 2048^2 map shared by the items; radius 0, 1 and 3; softness 0
and 0.01.  Each map is a field of random discs (occupancy 1, depths uniform).  For each case, alternating op and
restatement in --rounds rounds of --steps calls each (medians over the rounds):
  op_fwd_ms / op_fwd_bwd_ms        the public function through autograd, gradients to positions, matrix and map
  torch_fwd_ms / torch_fwd_bwd_ms  the same call with the restatement in its place (radius <= 1 only: at radius 3 its
                                   64 taps' intermediates do not fit in memory)
  kernel_fwd_ms / kernel_bwd_ms    the C ABI alone on preallocated buffers (backward: map memset, kernel, reduction)
  kernel_det_bwd_ms, det_scratch_mb  dirt_shadow_backward_deterministic on the same buffers, and its scratch
  *_bytes, *_of_peak               algorithmic bytes / kernel time, against the H100 SXM data sheet's 3.35 TB/s:
                                   fwd reads the positions and the map once and writes the visibility; bwd also reads
                                   grad_out and writes the position and map gradients
  reductions_per_point             the map-gradient reductions the warp aggregation leaves: per warp and tap, the number
                                   of distinct texels among its 32 lanes, over the points (computed from the lookups)
  op_held_mb / torch_held_mb       device memory autograd holds between forward and backward (output included)
CUDA events on the launching stream.  One JSON object with the card's name and power limit.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lightbench import PEAK_TBS, card, compare, held_mb, timed   # noqa: E402

B, SIDE = 64, 512


def make_map(items, S, gen):
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, S, device='cuda'), torch.linspace(-1, 1, S, device='cuda'),
                            indexing='ij')
    occ = torch.zeros((items, S, S), device='cuda')
    depth = torch.zeros((items, S, S), device='cuda')
    for _ in range(12):
        cx, cy = torch.rand((2, items, 1, 1), device='cuda', generator=gen) * 1.6 - 0.8
        rad = torch.rand((items, 1, 1), device='cuda', generator=gen) * 0.2 + 0.05
        z = torch.rand((items, 1, 1), device='cuda', generator=gen) * 0.5 - 0.5
        disc = ((xx - cx) ** 2 + (yy - cy) ** 2 < rad ** 2)
        occ = torch.where(disc, 1., occ)
        depth = torch.where(disc, z.expand_as(depth), depth)
    return torch.stack([occ, depth], -1)


def reductions_per_point(positions, S, R):
    """Distinct texels per warp and tap (the reductions left after MATCH.ANY), per point; the light matrix is the
    identity, so positions are light-clip coordinates."""
    p = positions.reshape(-1, 3)
    X, Yd = (p[:, 0] + 1) * (0.5 * S), (1 - p[:, 1]) * (0.5 * S)
    c0, r0 = torch.floor(X - 0.5).long(), torch.floor(Yd - 0.5).long()
    total = 0
    for i in range(2 * R + 2):
        for k in range(2 * R + 2):
            key = (r0 - R + i).clamp(0, S - 1) * S + (c0 - R + k).clamp(0, S - 1)
            key = key.reshape(-1, 32).sort(1).values
            total += int((key[:, 1:] != key[:, :-1]).sum()) + key.shape[0]
    return total / p.shape[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('shadowbench needs a CUDA device')
    from dirt_b200 import _lib, lighting
    gen = torch.Generator(device='cuda').manual_seed(0)
    N = SIDE * SIDE
    g = torch.linspace(-0.9, 0.9, SIDE, device='cuda')
    yy, xx = torch.meshgrid(g, g, indexing='ij')
    positions = torch.stack([xx.expand(B, SIDE, SIDE), yy.expand(B, SIDE, SIDE),
                             torch.rand((B, SIDE, SIDE), device='cuda', generator=gen) * 0.6 - 0.3], -1).reshape(B, N, 3)
    grad_out = torch.randn((B, N, 1), device='cuda', generator=gen)
    maps = {'per_item_1024': (make_map(B, 1024, gen), torch.eye(4, device='cuda').expand(B, 4, 4).contiguous()),
            'shared_2048': (make_map(1, 2048, gen)[0], torch.eye(4, device='cuda'))}
    L = _lib.lib()
    stream = torch.cuda.current_stream().cuda_stream
    results = {'card': card(), 'B': B, 'points_per_item': N, 'cases': []}
    for map_name, (smap, M) in maps.items():
        S = smap.shape[-2]
        per_item = smap.dim() == 4
        map_bytes = smap.numel() * 4
        for R in (0, 1, 3):
            for softness in (0., 0.01):
                case = {'map': map_name, 'radius': R, 'softness': softness}
                pos = positions.clone().requires_grad_(True)
                Mg = M.clone().requires_grad_(True)
                mg = smap.clone().requires_grad_(True)

                def op_fwd():
                    with torch.no_grad():
                        return lighting.shadow_visibility(positions, M, smap, R, softness, 0.005)

                def op_fwd_bwd():
                    (lighting.shadow_visibility(pos, Mg, mg, R, softness, 0.005) * grad_out).sum().backward()

                def ref_fwd():
                    with torch.no_grad():
                        return lighting._shadow_visibility(positions, M, smap, R, softness, 0.005)

                def ref_fwd_bwd():
                    (lighting._shadow_visibility(pos, Mg, mg, R, softness, 0.005) * grad_out).sum().backward()

                if R <= 1:
                    case['op_fwd_ms'], case['torch_fwd_ms'] = compare(op_fwd, ref_fwd, args.steps, args.rounds)
                    case['op_fwd_bwd_ms'], case['torch_fwd_bwd_ms'] = compare(op_fwd_bwd, ref_fwd_bwd, args.steps,
                                                                              args.rounds)
                    case['torch_held_mb'] = held_mb(lambda: lighting._shadow_visibility(pos, Mg, mg, R, softness, 0.005))
                else:
                    case['op_fwd_ms'] = sorted(timed(op_fwd, args.steps) for _ in range(args.rounds))[args.rounds // 2]
                    case['op_fwd_bwd_ms'] = sorted(timed(op_fwd_bwd, args.steps)
                                                   for _ in range(args.rounds))[args.rounds // 2]
                case['op_held_mb'] = held_mb(lambda: lighting.shadow_visibility(pos, Mg, mg, R, softness, 0.005))

                out = torch.empty((B * N,), device='cuda')
                gp = torch.empty((B * N, 3), device='cuda')
                gM = torch.empty(M.shape, device='cuda')
                gmap = torch.empty(smap.shape, device='cuda')
                ws = torch.empty(int(L.dirt_shadow_workspace_bytes(B, N)), dtype=torch.uint8, device='cuda')
                a = (positions.data_ptr(), 3, M.data_ptr(), smap.data_ptr(), int(per_item), S, S, R, softness, 0.005)
                go = grad_out.contiguous()

                def kfwd():
                    assert L.dirt_shadow_forward(*a, out.data_ptr(), B, N, stream) == 0

                def kbwd():
                    assert L.dirt_shadow_backward(*a, go.data_ptr(), gp.data_ptr(), gM.data_ptr(), gmap.data_ptr(),
                                                  ws.data_ptr(), ws.numel(), B, N, stream) == 0

                sb = int(L.dirt_shadow_backward_deterministic_bytes(B, N, int(per_item), S, S))
                scratch = torch.empty(sb, dtype=torch.uint8, device='cuda')

                def kdet():
                    assert L.dirt_shadow_backward_deterministic(*a, go.data_ptr(), gp.data_ptr(), gM.data_ptr(),
                                                                gmap.data_ptr(), ws.data_ptr(), ws.numel(),
                                                                scratch.data_ptr(), sb, B, N, stream) == 0

                case['kernel_fwd_ms'] = sorted(timed(kfwd, args.steps) for _ in range(args.rounds))[args.rounds // 2]
                case['kernel_bwd_ms'] = sorted(timed(kbwd, args.steps) for _ in range(args.rounds))[args.rounds // 2]
                case['kernel_det_bwd_ms'] = sorted(timed(kdet, args.steps) for _ in range(args.rounds))[args.rounds // 2]
                case['det_scratch_mb'] = sb / 2 ** 20
                del scratch
                fwd_bytes = B * N * (12 + 4) + map_bytes
                bwd_bytes = B * N * (12 + 4 + 12) + 2 * map_bytes
                case['fwd_bytes'], case['bwd_bytes'] = fwd_bytes, bwd_bytes
                case['fwd_of_peak'] = fwd_bytes / (case['kernel_fwd_ms'] * 1e-3) / (PEAK_TBS * 1e12)
                case['bwd_of_peak'] = bwd_bytes / (case['kernel_bwd_ms'] * 1e-3) / (PEAK_TBS * 1e12)
                case['reductions_per_point'] = reductions_per_point(positions, S, R)
                case['taps_per_point'] = (2 * R + 2) ** 2
                print(json.dumps(case), flush=True)
                results['cases'].append(case)
                del pos, Mg, mg
                torch.cuda.empty_cache()
    text = json.dumps(results, indent=1)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(text + '\n')
    print(text)


if __name__ == '__main__':
    main()
