"""Times the mipmapped cube-map lookup (dirt_b200.sample_cubemap(..., 'trilinear', lod=...)) against its torch
restatement (tests/cubemap_mip_restatement.py) and against the bilinear lookup.

    python profiles/cubemipbench.py [--steps 10] [--rounds 3] [--out FILE]

Workloads: N = 64 x 512^2 lookups, C = 3, into one shared cube map of 6 x 256^2 (L = 9) and one of 6 x 1024^2 (L = 11),
directions `reflection` and `random` (profiles/cubebench.py's), and lod patterns `sharp` (0), `glossy` (uniform in
[2, 5]) and `rough` (uniform in [L-3, L-1]).  For each, in --rounds alternating rounds of --steps calls (medians):
  op_fwd_ms / op_fwd_bwd_ms          the public function through autograd, gradients to cube map, directions and lod
  bilinear_fwd_ms / bilinear_fwd_bwd_ms  sample_cubemap(..., 'bilinear') on the same directions
  torch_fwd_ms / torch_fwd_bwd_ms    the restatement, and op_small_* the op, on the first RESTATEMENT_IMAGES images
                                     only (the restatement of all 64 holds more than the card's memory)
  kernel_fwd_ms                      dirt_cubemap_sample_trilinear on preallocated buffers (pyramid and atlases included)
  build_ms                           dirt_cubemap_sample_trilinear of one lookup: the pyramid and the atlases
  kernel_bwd_ms / kernel_bwd_det_ms  dirt_cubemap_sample_trilinear_backward, every gradient, default / deterministic
  kernel_bwd_no_smem_ms              (rough only) the default backward of a build with DIRT_CUBE_MIP_SMEM_FLOATS=0,
                                     compiled by this script into a temporary directory
  *_bytes, *_of_peak                 algorithmic bytes / kernel time, against the H100 SXM data sheet's 3.35 TB/s
  op_held_mb                         device memory autograd holds between forward and backward (output included)
CUDA events on the launching stream.  One JSON object with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'profiles'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from cubebench import directions  # noqa: E402
from lightbench import PEAK_TBS, card, compare, held_mb, timed  # noqa: E402
import cubemap_mip_restatement as cmm  # noqa: E402
import cubemap_restatement as cm  # noqa: E402

RESTATEMENT_IMAGES = 4


def levels(S):
    return cmm.level_count(S)


def atlas_floats(S, C):
    return sum(6 * ((S >> k) + 2) ** 2 * C for k in range(levels(S)))


def algorithmic_bytes(N, S, C):
    """fwd: read the cube map, write and read the pyramid (1/3 of it), write the atlases, read the directions and lod,
    write the output.  bwd: read directions, lod and grad_out, write grad_directions and grad_lod; zero, then read the
    atlas gradients, write and read the pyramid's gradient, read and write grad_cubemap.  Texel reads by the lookups
    are counted once, as the atlases' size."""
    cube, atlas = 4 * 6 * S * S * C, 4 * atlas_floats(S, C)
    pyr = cube // 3
    fwd = cube + 2 * pyr + 2 * atlas + 4 * N * (3 + 1 + C)
    bwd = 4 * N * (3 + 1 + C + 3 + 1) + 2 * atlas + 2 * pyr + 3 * cube
    return fwd, bwd


def no_smem_library(tmp):
    from dirt_b200 import _lib, build
    out = os.path.join(tmp, 'libdirt_b200_cube_mip_no_smem.so')
    srcs = [os.path.join(ROOT, 'dirt_b200', 'csrc', s) for s in build.SOURCES]
    cmd = [build._nvcc()] + build.NVCC_FLAGS + ['-DDIRT_CUBE_MIP_SMEM_FLOATS=0', '-o', out] + srcs
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise SystemExit(proc.stdout + proc.stderr)
    return _lib.load(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('cubemipbench.py needs a CUDA device')
    import dirt_b200 as dirt
    from dirt_b200 import _lib
    L = _lib.lib()
    tmp = tempfile.mkdtemp(prefix='cubemipbench_')
    plain = no_smem_library(tmp)
    dev = torch.device('cuda', 0)
    B, H, W, C = 64, 512, 512, 3
    N = H * W
    name, limit = card()
    result = {'device': name, 'power_limit': limit, 'lookups': B * N, 'channels': C, 'steps': args.steps,
              'rounds': args.rounds, 'restatement_images': RESTATEMENT_IMAGES, 'cases': []}
    g = torch.Generator(device=dev).manual_seed(0)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    grad_out = torch.randn(B, N, C, generator=g, device=dev)
    for S in (256, 1024):
        Lv = levels(S)
        cube = torch.rand(6, S, S, C, generator=g, device=dev)
        for k in range(Lv):
            cm.border_table(S >> k)   # built once per size, outside the timed window
        for pattern in ('reflection', 'random'):
            dirs = directions(pattern, B, H, W, dev, g)
            for lod_pattern in ('sharp', 'glossy', 'rough'):
                if lod_pattern == 'sharp':
                    lod = torch.zeros(B, N, device=dev)
                elif lod_pattern == 'glossy':
                    lod = torch.rand(B, N, generator=g, device=dev) * 3 + 2
                else:
                    lod = torch.rand(B, N, generator=g, device=dev) * 2 + (Lv - 3)
                leaves = [cube.clone().requires_grad_(True), dirs.clone().requires_grad_(True),
                          lod.clone().requires_grad_(True)]
                small = [cube.clone().requires_grad_(True), dirs[:RESTATEMENT_IMAGES].clone().requires_grad_(True),
                         lod[:RESTATEMENT_IMAGES].clone().requires_grad_(True)]
                op = lambda c, x, lo: dirt.sample_cubemap(c, x, 'trilinear', lod=lo)
                bil = lambda c, x, lo: dirt.sample_cubemap(c, x, 'bilinear')

                def fwd(fn, vs):
                    with torch.no_grad():
                        return fn(*vs)

                def fwd_bwd(fn, vs, go):
                    for v in vs:
                        v.grad = None
                    fn(*vs).backward(go)

                atlas = torch.empty(int(L.dirt_cubemap_mip_atlas_bytes(1, S, C)) // 4, device=dev)
                out = torch.empty(B, N, C, device=dev)
                gc, gd, gl = torch.empty_like(cube), torch.empty_like(dirs), torch.empty_like(lod)
                scratch = {det: torch.empty(int(L.dirt_cubemap_sample_trilinear_backward_bytes(1, S, C, B, N, det)),
                                            dtype=torch.uint8, device=dev) for det in (0, 1)}
                run_fwd = lambda: L.dirt_cubemap_sample_trilinear(p(cube), p(dirs), p(lod), p(atlas), p(out), 1, S, C, B,
                                                                  N, stream())
                run_build = lambda: L.dirt_cubemap_sample_trilinear(p(cube), p(dirs), p(lod), p(atlas), p(out), 1, S, C,
                                                                    1, 1, stream())

                def bwd(lib, det):
                    return lambda: lib.dirt_cubemap_sample_trilinear_backward(
                        p(atlas), p(dirs), p(lod), p(grad_out), p(gc), p(gd), p(gl), 1, S, C, B, N, det,
                        p(scratch[det]), scratch[det].numel(), stream())
                assert run_fwd() == 0
                fns = [run_fwd, run_build, bwd(L, 0), bwd(L, 1)] + ([bwd(plain, 0)] if lod_pattern == 'rough' else [])
                times = [[] for _ in fns]
                for _ in range(args.rounds):
                    for t, fn in zip(times, fns):
                        t.append(timed(fn, args.steps))
                med = [statistics.median(t) for t in times]
                k_fwd, k_build, k_bwd, k_det = med[:4]
                op_fwd, bil_fwd = compare(lambda: fwd(op, leaves), lambda: fwd(bil, leaves), args.steps, args.rounds)
                op_fb, bil_fb = compare(lambda: fwd_bwd(op, leaves, grad_out), lambda: fwd_bwd(bil, leaves, grad_out),
                                        args.steps, args.rounds)
                go_small = grad_out[:RESTATEMENT_IMAGES]
                small_fwd, torch_fwd = compare(lambda: fwd(op, small), lambda: fwd(cmm.sample, small), args.steps,
                                               args.rounds)
                small_fb, torch_fb = compare(lambda: fwd_bwd(op, small, go_small),
                                             lambda: fwd_bwd(cmm.sample, small, go_small), args.steps, args.rounds)
                fb, bb = algorithmic_bytes(B * N, S, C)
                row = {'case': '%s, %s, 6 x %d^2' % (pattern, lod_pattern, S), 'levels': Lv,
                       'op_fwd_ms': op_fwd, 'op_fwd_bwd_ms': op_fb, 'bilinear_fwd_ms': bil_fwd,
                       'bilinear_fwd_bwd_ms': bil_fb, 'op_small_fwd_ms': small_fwd, 'torch_fwd_ms': torch_fwd,
                       'op_small_fwd_bwd_ms': small_fb, 'torch_fwd_bwd_ms': torch_fb,
                       'kernel_fwd_ms': k_fwd, 'build_ms': k_build, 'kernel_bwd_ms': k_bwd, 'kernel_bwd_det_ms': k_det,
                       'fwd_bytes': fb, 'bwd_bytes': bb,
                       'kernel_fwd_of_peak': fb / (k_fwd * 1e-3) / 1e12 / PEAK_TBS,
                       'kernel_bwd_of_peak': bb / (k_bwd * 1e-3) / 1e12 / PEAK_TBS,
                       'op_held_mb': held_mb(lambda: op(*leaves)),
                       'speedup_fwd_small': torch_fwd / small_fwd, 'speedup_fwd_bwd_small': torch_fb / small_fb}
                if lod_pattern == 'rough':
                    row['kernel_bwd_no_smem_ms'] = med[4]
                result['cases'].append(row)
                print(json.dumps(row), flush=True)
                del leaves, small, atlas, out, gc, gd, gl, scratch
                torch.cuda.empty_cache()
            del dirs
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            f.write(json.dumps(result, indent=1) + '\n')


if __name__ == '__main__':
    main()
