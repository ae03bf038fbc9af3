"""Times the reflectance models' CUDA path against their torch restatement (dirt_b200/lighting.py).

    python profiles/lightbench.py [--steps 20] [--rounds 3] [--out FILE]

Workloads: each model alone on N = 64 x 512^2 points, C = 3, contiguous [N, 3] inputs and parameters shared by all
points (the call pattern of the example shaders); and examples/deferred.py's shader_fn on a 64 x 512 x 512 x 10
G-buffer (its per-point inputs are strided slices of the G-buffer).  For each, alternating op and restatement in
--rounds rounds of --steps calls each (the figures are the median over the rounds):
  op_fwd_ms / op_fwd_bwd_ms        the public function through autograd (Python layer and allocations included)
  torch_fwd_ms / torch_fwd_bwd_ms  the same call with the restatement in its place
  kernel_fwd_ms / kernel_bwd_ms    the C ABI alone on preallocated buffers (backward: every gradient), models only
  *_bytes, *_of_peak               algorithmic bytes from shapes / kernel time, against the H100 SXM data sheet's 3.35 TB/s
  op_held_mb / torch_held_mb       device memory autograd holds between forward and backward (output included)
CUDA events on the launching stream.  One JSON object with the card's name and power limit.
"""
import argparse
import ctypes
import importlib.util
import inspect
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PEAK_TBS = 3.35   # H100 SXM data sheet HBM3 bandwidth
MODELS = ['diffuse_directional', 'specular_directional', 'diffuse_point']
ARGS = {'diffuse_directional': ['nrm', 'col', 'ldir', 'lcol'],
        'specular_directional': ['pos', 'nrm', 'col', 'ldir', 'lcol', 'cam', 'shin'],
        'diffuse_point': ['pos', 'nrm', 'col', 'lpos', 'lcol']}


def algorithmic_bytes(model, N, C):
    """fwd: read the per-point inputs once, write the output.  bwd: read the per-point inputs and grad_out, write every
    per-point gradient (the parameter gradients and partials are negligible)."""
    k = 3 + C + (3 if model != 'diffuse_directional' else 0)
    return 4 * N * (k + C), 4 * N * (k + C + k)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = 'unknown'
    return name, limit


def timed(fn, steps, warmup=2):
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


def held_mb(fn):
    """Device memory allocated after the forward call, while its graph is alive, minus that before it."""
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated() - before
    del out
    return held / 2 ** 20


def compare(op, ref, steps, rounds):
    """Median times of op and ref over `rounds` alternating rounds, each `steps` calls."""
    a, b = [], []
    for _ in range(rounds):
        a.append(timed(op, steps))
        b.append(timed(ref, steps))
    return statistics.median(a), statistics.median(b)


def restatement(lighting, model):
    """A stand-in for lighting.<model> that always runs the torch restatement (same signature and conversions)."""
    signature = inspect.signature(getattr(lighting, model))

    def fn(*args, **kwargs):
        bound = signature.bind(*args, **kwargs)
        bound.apply_defaults()
        values = dict(bound.arguments)
        values.pop('name')
        double_sided = values.pop('double_sided')
        dev = next(iter(values.values())).device
        return getattr(lighting, '_' + model)(*[torch.as_tensor(v, dtype=torch.float32, device=dev)
                                                for v in values.values()], double_sided)
    return fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('lightbench.py needs a CUDA device')
    from dirt_b200 import _lib, lighting
    L = _lib.lib()
    dev = torch.device('cuda', 0)
    B, H, W, C = 64, 512, 512, 3
    N = B * H * W
    name, limit = card()
    result = {'device': name, 'power_limit': limit, 'points': N, 'channels': C, 'steps': args.steps,
              'rounds': args.rounds, 'cases': []}
    g = torch.Generator(device=dev).manual_seed(0)
    x = dict(pos=torch.rand(N, 3, generator=g, device=dev) * 4 - 2,
             nrm=torch.nn.functional.normalize(torch.randn(N, 3, generator=g, device=dev), dim=-1),
             col=torch.rand(N, C, generator=g, device=dev),
             ldir=torch.nn.functional.normalize(torch.tensor([1., -0.3, -0.5], device=dev), dim=0),
             lcol=torch.ones(C, device=dev), lpos=torch.tensor([3., 4., 5.], device=dev),
             cam=torch.tensor([0., 1.5, 6.], device=dev), shin=torch.tensor(6., device=dev))
    grad_out = torch.randn(N, C, generator=g, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for mi, model in enumerate(MODELS):
        keys = ARGS[model]
        leaves = {k: x[k].clone().requires_grad_(True) for k in keys}
        op_fn, ref_fn = getattr(lighting, model), restatement(lighting, model)

        def fwd(fn):
            with torch.no_grad():
                return fn(*[x[k] for k in keys])

        def fwd_bwd(fn):
            for v in leaves.values():
                v.grad = None
            fn(*[leaves[k] for k in keys]).backward(grad_out)

        # the ABI on preallocated buffers
        has_pos = model != 'diffuse_directional'
        light = x['lpos'] if model == 'diffuse_point' else x['ldir']
        sp = model == 'specular_directional'
        inputs = [mi, 1, p(x['nrm']), 3, p(x['pos'] if has_pos else None), 3, p(x['col']), C, p(light), 0, p(x['lcol']),
                  0, p(x['cam'] if sp else None), 0, p(x['shin'] if sp else None), 0]
        out = torch.empty(N, C, device=dev)
        grads = [torch.empty(N, 3, device=dev), torch.empty(N, 3, device=dev) if has_pos else None,
                 torch.empty(N, C, device=dev), torch.empty(3, device=dev), torch.empty(C, device=dev),
                 torch.empty(3, device=dev) if sp else None, torch.empty(1, device=dev) if sp else None]
        ws_bytes = int(L.dirt_lighting_workspace_bytes(1, N, C))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        k_fwd = timed(lambda: L.dirt_lighting_forward(*inputs, p(out), 1, N, C, stream()), args.steps)
        k_bwd = timed(lambda: L.dirt_lighting_backward(*inputs, p(grad_out), *[p(t) for t in grads], p(ws), ws_bytes, 1,
                                                       N, C, stream()), args.steps)
        op_fwd, torch_fwd = compare(lambda: fwd(op_fn), lambda: fwd(ref_fn), args.steps, args.rounds)
        op_fb, torch_fb = compare(lambda: fwd_bwd(op_fn), lambda: fwd_bwd(ref_fn), args.steps, args.rounds)
        fb, bb = algorithmic_bytes(model, N, C)
        case = {'case': model, 'op_fwd_ms': op_fwd, 'torch_fwd_ms': torch_fwd, 'op_fwd_bwd_ms': op_fb,
                'torch_fwd_bwd_ms': torch_fb, 'kernel_fwd_ms': k_fwd, 'kernel_bwd_ms': k_bwd, 'fwd_bytes': fb,
                'bwd_bytes': bb,
                'kernel_fwd_of_peak': fb / (k_fwd * 1e-3) / 1e12 / PEAK_TBS,
                'kernel_bwd_of_peak': bb / (k_bwd * 1e-3) / 1e12 / PEAK_TBS,
                'op_held_mb': held_mb(lambda: op_fn(*[leaves[k] for k in keys])),
                'torch_held_mb': held_mb(lambda: ref_fn(*[leaves[k] for k in keys]))}
        case['speedup_fwd'] = torch_fwd / op_fwd
        case['speedup_fwd_bwd'] = torch_fb / op_fb
        result['cases'].append(case)
        print(json.dumps(case), flush=True)
        del leaves, out, grads, ws
        torch.cuda.empty_cache()

    # examples/deferred.py's shader on a cfg3-sized G-buffer
    spec = importlib.util.spec_from_file_location('deferred_example', os.path.join(ROOT, 'examples', 'deferred.py'))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    from dirt_b200 import matrices
    gbuffer = torch.rand(B, H, W, 10, generator=g, device=dev)
    gbuffer[..., 7:] = torch.nn.functional.normalize(gbuffer[..., 7:] - 0.5, dim=-1)
    view = matrices.compose(matrices.translation([0., -1.5, -3.5]), matrices.rodrigues([-0.3, 0., 0.])).to(dev)
    light = x['ldir'].clone().requires_grad_(True)
    gb = gbuffer.clone().requires_grad_(True)
    shade_grad = torch.randn(B, H, W, 3, generator=g, device=dev)
    cuda_fns = (lighting.diffuse_directional, lighting.specular_directional)
    torch_fns = (restatement(lighting, 'diffuse_directional'), restatement(lighting, 'specular_directional'))

    def use(fns):
        lighting.diffuse_directional, lighting.specular_directional = fns

    def shader_fwd(fns):
        use(fns)
        with torch.no_grad():
            return ex.shader_fn(gbuffer, view, x['ldir'])

    def shader_fwd_bwd(fns):
        use(fns)
        gb.grad, light.grad = None, None
        ex.shader_fn(gb, view, light).backward(shade_grad)

    def shader_held(fns):
        use(fns)
        return held_mb(lambda: ex.shader_fn(gb, view, light))

    op_fwd, torch_fwd = compare(lambda: shader_fwd(cuda_fns), lambda: shader_fwd(torch_fns), args.steps, args.rounds)
    op_fb, torch_fb = compare(lambda: shader_fwd_bwd(cuda_fns), lambda: shader_fwd_bwd(torch_fns), args.steps,
                              args.rounds)
    case = {'case': 'deferred shader_fn', 'op_fwd_ms': op_fwd, 'torch_fwd_ms': torch_fwd, 'op_fwd_bwd_ms': op_fb,
            'torch_fwd_bwd_ms': torch_fb, 'op_held_mb': shader_held(cuda_fns), 'torch_held_mb': shader_held(torch_fns),
            'speedup_fwd': torch_fwd / op_fwd, 'speedup_fwd_bwd': torch_fb / op_fb}
    use(cuda_fns)
    result['cases'].append(case)
    print(json.dumps(case), flush=True)
    print(json.dumps(result))
    if args.out:
        with open(args.out, 'w') as f:
            f.write(json.dumps(result, indent=1) + '\n')


if __name__ == '__main__':
    main()
