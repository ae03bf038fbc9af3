"""Times the triangle-setup kernel of one or more prebuilt variants of libdirt_b200.so, next to the step it sits in.

    python profiles/setupbench.py [--workloads cfg3,cfg4,cfg5,cube] [--steps 30] [--rounds 3] lib_a.so lib_b.so ...
                                  [--setup-only lib_c.so ...]

Each library is loaded in its own process (DIRT_B200_LIB) and run through bench.PreparedStep on every workload in turn
(seed 1, as kbench.py): the setup kernel alone and the raster kernel alone through the library's timer hooks (ids 3 and 1),
the forward call, the backward call (the forward's workspace handed back, as in the bench step) and the graph-replayed
step, each averaged over --steps calls.  Libraries listed after --setup-only are timing builds (DIRT_SETUP_ABLATE) whose
forward call runs the setup kernel alone: only the setup kernel and the forward call are timed for them.
The libraries are run in turn, --rounds times over, so that a drift of the card shows up in every variant alike.  One JSON
line per (round, library), with the card's name, power limit and maximum SM clock as nvidia-smi reports them.
Variants are built with `python profiles/build_variant.py TAG -DFLAG=...` (dirt_b200/variants/, git-ignored .so files).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(',')]
        return {'gpu': name, 'power_limit': power, 'sm_clock_max': clock}
    except Exception as e:   # said in the line, not guessed
        return {'gpu': 'unknown (%s)' % type(e).__name__}


def one(args):
    sys.path.insert(0, ROOT)
    import torch
    import bench
    from dirt_b200 import scenes
    device = torch.device('cuda', 0)
    n = args.steps
    res = {}
    for workload in args.workloads.split(','):
        gen, kwargs, _ = bench.WORKLOADS[workload]
        kwargs = dict(kwargs)
        if workload != 'cfg2':
            kwargs['seed'] = 1
        prep = bench.PreparedStep(getattr(scenes, gen)(**kwargs), device)
        for _ in range(3):
            prep.forward() if args.timing_build else prep.local_step(0)
        torch.cuda.synchronize()

        def timed(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(n):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / n

        def kernel(which, fn):
            prep.lib.dirt_kernel_timer_enable(which)
            total = 0.0
            for _ in range(n):
                fn()
                total += float(prep.lib.dirt_kernel_timer_elapsed_ms())
            prep.lib.dirt_kernel_timer_enable(0)
            return total / n

        r = {'setup_kernel_ms': kernel(3, prep.forward), 'forward_call_ms': timed(prep.forward)}
        if not args.timing_build:
            r['raster_kernel_ms'] = kernel(1, prep.forward)
            prep.forward()
            r['backward_call_ms'] = timed(prep.backward)
            prep.capture()
            r['graph_step_ms'] = timed(lambda: prep.graphs[0].replay())
        res[workload] = {k: round(v, 5) for k, v in r.items()}
        del prep
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    out = {'lib': os.path.basename(os.environ.get('DIRT_B200_LIB', 'default')), 'round': args.round, 'steps': n}
    out.update(card())
    out['workloads'] = res
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('libs', nargs='*')
    ap.add_argument('--setup-only', nargs='*', default=[], metavar='LIB')
    ap.add_argument('--workloads', default='cfg3,cfg4,cfg5,cube')
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--round', type=int, default=0)
    ap.add_argument('--one', action='store_true')
    ap.add_argument('--timing-build', action='store_true')
    args = ap.parse_args()
    if args.one:
        return one(args)
    libs = [(l, False) for l in (args.libs or [os.path.join(ROOT, 'dirt_b200', 'libdirt_b200.so')])]
    libs += [(l, True) for l in args.setup_only]
    for rnd in range(args.rounds):
        for lib, setup_only in libs:
            env = dict(os.environ, DIRT_B200_LIB=os.path.abspath(lib))
            cmd = [sys.executable, os.path.abspath(__file__), '--one', '--workloads', args.workloads, '--steps', str(args.steps),
                   '--round', str(rnd)] + (['--timing-build'] if setup_only else [])
            proc = subprocess.run(cmd, env=env, capture_output=True, text=True)
            line = [l for l in proc.stdout.splitlines() if l.startswith('{')]
            print(line[-1] if line else json.dumps({'lib': os.path.basename(lib), 'round': rnd,
                                                    'error': (proc.stderr or proc.stdout)[-400:]}), flush=True)


if __name__ == '__main__':
    main()
