"""Times the GGX specular model's CUDA path against its torch restatement (dirt_b200/lighting.py).

    python profiles/ggxbench.py [--steps 20] [--rounds 3] [--out FILE]

Workloads: each light kind alone on N = 64 x 512^2 points, C = 3, contiguous [N, k] inputs, with the light, its colour
and the camera shared by all points and one per item; and a deferred shader, diffuse_directional + specular_ggx_directional
on a 64 x 512 x 512 x 13 G-buffer [position, normal, albedo, roughness, specular colour], each input a strided slice of
it.  For each, alternating op and restatement in --rounds rounds of --steps calls each (medians over the rounds):
  op_fwd_ms / op_fwd_bwd_ms        the public function through autograd (Python layer and allocations included)
  torch_fwd_ms / torch_fwd_bwd_ms  the same call with the restatement in its place
  kernel_fwd_ms / kernel_bwd_ms    the C ABI alone on preallocated buffers (backward: every gradient), models only
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
sys.path.insert(0, os.path.join(ROOT, 'profiles'))
from lightbench import PEAK_TBS, card, compare, held_mb, timed   # noqa: E402

KEYS = ['pos', 'nrm', 'rough', 'spec', 'light', 'lcol', 'cam']


def algorithmic_bytes(N, C):
    """fwd: read positions, normals, roughness and F0 once, write the output.  bwd: read them and grad_out, write every
    per-point gradient (the parameter gradients and partials are negligible)."""
    k = 3 + 3 + 1 + C
    return 4 * N * (k + C), 4 * N * (k + C + k)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('ggxbench.py needs a CUDA device')
    from dirt_b200 import _lib, lighting
    L = _lib.lib()
    dev = torch.device('cuda', 0)
    B, H, W, C = 64, 512, 512, 3
    V = H * W
    N = B * V
    name, limit = card()
    result = {'device': name, 'power_limit': limit, 'points': N, 'channels': C, 'steps': args.steps,
              'rounds': args.rounds, 'cases': []}
    g = torch.Generator(device=dev).manual_seed(0)
    x = dict(pos=torch.rand(B, V, 3, generator=g, device=dev) * 4 - 2,
             nrm=torch.nn.functional.normalize(torch.randn(B, V, 3, generator=g, device=dev), dim=-1),
             rough=torch.rand(B, V, 1, generator=g, device=dev) * 0.9 + 0.05,
             spec=torch.rand(B, V, C, generator=g, device=dev))
    grad_out = torch.randn(B, V, C, generator=g, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for point in (False, True):
        for per_item in (False, True):
            light = torch.tensor([3., 4., 5.], device=dev) if point else \
                torch.nn.functional.normalize(torch.tensor([1., -0.3, -0.5], device=dev), dim=0)
            params = dict(light=light, lcol=torch.ones(C, device=dev), cam=torch.tensor([0., 1.5, 6.], device=dev))
            if per_item:
                params = {k: v.expand(B, -1).contiguous() for k, v in params.items()}
            y = dict(x, **params)
            leaves = {k: y[k].clone().requires_grad_(True) for k in KEYS}
            op_fn = lighting.specular_ggx_point if point else lighting.specular_ggx_directional
            ref_fn = lambda *t: lighting._specular_ggx(*t, point, False)

            def fwd(fn):
                with torch.no_grad():
                    return fn(*[y[k] for k in KEYS])

            def fwd_bwd(fn):
                for v in leaves.values():
                    v.grad = None
                fn(*[leaves[k] for k in KEYS]).backward(grad_out)

            # the ABI on preallocated buffers
            flag = int(per_item)
            inputs = [int(point), 0, p(y['nrm']), 3, p(y['pos']), 3, p(y['rough']), 1, p(y['spec']), C, p(y['light']),
                      flag, p(y['lcol']), flag, p(y['cam']), flag]
            out = torch.empty(N, C, device=dev)
            grads = [torch.empty(N, 3, device=dev), torch.empty(N, 3, device=dev), torch.empty(N, device=dev),
                     torch.empty(N, C, device=dev)] + [torch.empty_like(params[k]) for k in ('light', 'lcol', 'cam')]
            ws_bytes = int(L.dirt_lighting_workspace_bytes(B, V, C))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            k_fwd = timed(lambda: L.dirt_ggx_lighting_forward(*inputs, p(out), B, V, C, stream()), args.steps)
            k_bwd = timed(lambda: L.dirt_ggx_lighting_backward(*inputs, p(grad_out), *[p(t) for t in grads], p(ws),
                                                               ws_bytes, B, V, C, stream()), args.steps)
            op_fwd, torch_fwd = compare(lambda: fwd(op_fn), lambda: fwd(ref_fn), args.steps, args.rounds)
            op_fb, torch_fb = compare(lambda: fwd_bwd(op_fn), lambda: fwd_bwd(ref_fn), args.steps, args.rounds)
            fb, bb = algorithmic_bytes(N, C)
            case = {'case': '%s, %s parameters' % ('point' if point else 'directional',
                                                   'per-item' if per_item else 'shared'),
                    'op_fwd_ms': op_fwd, 'torch_fwd_ms': torch_fwd, 'op_fwd_bwd_ms': op_fb,
                    'torch_fwd_bwd_ms': torch_fb, 'kernel_fwd_ms': k_fwd, 'kernel_bwd_ms': k_bwd, 'fwd_bytes': fb,
                    'bwd_bytes': bb,
                    'kernel_fwd_of_peak': fb / (k_fwd * 1e-3) / 1e12 / PEAK_TBS,
                    'kernel_bwd_of_peak': bb / (k_bwd * 1e-3) / 1e12 / PEAK_TBS,
                    'op_held_mb': held_mb(lambda: op_fn(*[leaves[k] for k in KEYS])),
                    'torch_held_mb': held_mb(lambda: ref_fn(*[leaves[k] for k in KEYS]))}
            case['speedup_fwd'] = torch_fwd / op_fwd
            case['speedup_fwd_bwd'] = torch_fb / op_fb
            result['cases'].append(case)
            print(json.dumps(case), flush=True)
            del leaves, out, grads, ws
            torch.cuda.empty_cache()

    # a deferred shader: diffuse plus GGX from strided slices of one G-buffer
    del x, grad_out
    torch.cuda.empty_cache()
    gbuffer = torch.rand(B, H, W, 13, generator=g, device=dev)
    gbuffer[..., 3:6] = torch.nn.functional.normalize(gbuffer[..., 3:6] - 0.5, dim=-1)
    ldir = torch.nn.functional.normalize(torch.tensor([1., -0.3, -0.5], device=dev), dim=0)
    lcol, cam = torch.ones(C, device=dev), torch.tensor([0., 1.5, 6.], device=dev)
    gb = gbuffer.clone().requires_grad_(True)
    shade_grad = torch.randn(B, H, W, 3, generator=g, device=dev)
    ggx_ref = lambda *t: lighting._specular_ggx(*t, False, False)

    def shader(gbuf, ggx):
        s = lambda a, b: gbuf[..., a:b].reshape(B, -1, b - a)
        lit = lighting.diffuse_directional(s(3, 6), s(6, 9), ldir, lcol, False) + \
            ggx(s(0, 3), s(3, 6), s(9, 10), s(10, 13), ldir, lcol, cam)
        return lit.reshape(B, H, W, 3)

    def shader_fwd(ggx):
        with torch.no_grad():
            return shader(gbuffer, ggx)

    def shader_fwd_bwd(ggx):
        gb.grad = None
        shader(gb, ggx).backward(shade_grad)

    op_fwd, torch_fwd = compare(lambda: shader_fwd(lighting.specular_ggx_directional), lambda: shader_fwd(ggx_ref),
                                args.steps, args.rounds)
    op_fb, torch_fb = compare(lambda: shader_fwd_bwd(lighting.specular_ggx_directional),
                              lambda: shader_fwd_bwd(ggx_ref), args.steps, args.rounds)
    case = {'case': 'deferred diffuse + GGX', 'op_fwd_ms': op_fwd, 'torch_fwd_ms': torch_fwd, 'op_fwd_bwd_ms': op_fb,
            'torch_fwd_bwd_ms': torch_fb,
            'op_held_mb': held_mb(lambda: shader(gb, lighting.specular_ggx_directional)),
            'torch_held_mb': held_mb(lambda: shader(gb, ggx_ref)),
            'speedup_fwd': torch_fwd / op_fwd, 'speedup_fwd_bwd': torch_fb / op_fb}
    result['cases'].append(case)
    print(json.dumps(case), flush=True)
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            f.write(json.dumps(result, indent=1) + '\n')


if __name__ == '__main__':
    main()
