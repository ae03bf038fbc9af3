"""Times the backward kernel of one or more prebuilt variants of libdirt_b200.so, next to the call and the step it sits in;
with --census, counts on the CPU what the backward kernel's tiles hold.

    python profiles/bwdbench.py [--workloads cfg3,cfg4,cfg5,cube] [--steps 30] [--rounds 3] lib_a.so lib_b.so ...
    python profiles/bwdbench.py --census [--workloads ...] [--images 2]

Timing: each library is loaded in its own process (DIRT_B200_LIB) and run through bench.PreparedStep on every workload
in turn (seed 1, as kbench.py and setupbench.py): the backward kernel alone through the library's timer hook (id 2), the
backward call (the forward's workspace handed back, as in the bench step) and the graph-replayed step, each averaged over
--steps calls.  The libraries are run in turn, --rounds times over, so that a drift of the card shows up in every
variant alike.  One JSON line per (round, library), with the card's name, power limit and maximum SM clock as nvidia-smi
reports them.  Variants are built with `python profiles/build_variant.py TAG -DFLAG=...` (dirt_b200/variants/).

Census: the CPU oracle's face ids and dilation masks of the first --images images of each workload (the bench scenes,
seed 1), cut into the backward kernel's 8x8 tiles.  A tile goes past the coverage flag when its 16x8 forward tile or one
of that tile's 8 neighbours shows a face, and past the empty-tile exit when a face covers one of its 64 pixels or 32 ring
cells (the 10x10 halo without its corners).  For those tiles: distinct faces of tile + ring (the face-table slots,
against the 24 / 32 slots of C = 4 / C = 3), faces owning a tile pixel (the only slots with colour records), faces of the
ring only (slots that can hold position records only), faces all of whose tile pixels dilate away (colour records only,
unless a neighbour dilates into them), and, C = 4, the covered-or-near pixels whose two channel groups disagree on
dilating.  One JSON line per workload.
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


def scene_of(workload, batch=None):
    sys.path.insert(0, ROOT)
    import bench
    from dirt_b200 import scenes
    gen, kwargs, _ = bench.WORKLOADS[workload]
    kwargs = dict(kwargs)
    if workload != 'cfg2':
        kwargs['seed'] = 1
    if batch:
        kwargs['batch'] = batch
    return getattr(scenes, gen)(**kwargs)


def one(args):
    sys.path.insert(0, ROOT)
    import torch
    import bench
    device = torch.device('cuda', 0)
    n = args.steps
    res = {}
    for workload in args.workloads.split(','):
        prep = bench.PreparedStep(scene_of(workload), device)
        for _ in range(3):
            prep.local_step(0)
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

        prep.forward()
        prep.lib.dirt_kernel_timer_enable(2)
        total = 0.0
        for _ in range(n):
            prep.backward()
            total += float(prep.lib.dirt_kernel_timer_elapsed_ms())
        prep.lib.dirt_kernel_timer_enable(0)
        r = {'backward_kernel_ms': total / n, 'backward_call_ms': timed(prep.backward)}
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


def census(workload, images):
    import numpy as np
    sys.path.insert(0, ROOT)
    from oracle import oracle
    s = scene_of(workload)
    B = s['background'].shape[0]
    s = {k: (v[:images] if v.shape[0] == B else v) for k, v in s.items()}
    pixels, ids = oracle.forward(s['background'], s['vertices'], s['vertex_colors'], s['faces'], return_face_ids=True)
    C = pixels.shape[-1]
    gp = np.random.default_rng(0).standard_normal(pixels.shape).astype(np.float32)
    masks = oracle.backward(s['vertices'], s['faces'], pixels, gp, return_dilation=True)[3]
    nb, H, W = ids.shape
    ty, tx = (H + 7) // 8, (W + 7) // 8
    pad = -np.ones((nb, ty * 8 + 2, tx * 8 + 2), np.int32)
    pad[:, 1:H + 1, 1:W + 1] = ids
    halo = np.lib.stride_tricks.sliding_window_view(pad, (10, 10), axis=(1, 2))[:, ::8, ::8]   # [nb, ty, tx, 10, 10]
    inner = np.zeros((10, 10), bool)
    inner[1:9, 1:9] = True
    ring = ~inner
    ring[[0, 0, 9, 9], [0, 9, 0, 9]] = False
    tile_ids = halo[..., inner].reshape(nb, ty, tx, 64)
    ring_ids = halo[..., ring].reshape(nb, ty, tx, 32)
    # forward coverage flags: a 16x8 tile showing a face marks itself and its 8 neighbours
    fy, fx = (H + 7) // 8, (W + 15) // 16
    cov = np.zeros((nb, fy * 8, fx * 16), bool)
    cov[:, :H, :W] = ids >= 0
    shows = cov.reshape(nb, fy, 8, fx, 16).any(axis=(2, 4))
    sp = np.pad(shows, ((0, 0), (1, 1), (1, 1)))
    fflag = np.zeros_like(shows)
    for dy in (0, 1, 2):
        for dx in (0, 1, 2):
            fflag |= sp[:, dy:dy + fy, dx:dx + fx]
    flagged = np.repeat(fflag, 2, axis=2)[:, :, :tx]
    both = np.concatenate([tile_ids, ring_ids], axis=-1)
    live = flagged & (both >= 0).any(axis=-1)

    def distinct(a):
        a = np.sort(a, axis=-1)
        return (a[..., :1] >= 0).sum(-1) + ((a[..., 1:] != a[..., :-1]) & (a[..., 1:] >= 0)).sum(-1)

    n_all, n_tile = distinct(both)[live], distinct(tile_ids)[live]
    # faces all of whose tile pixels dilate away in the first channel group
    dil = np.zeros((nb, ty * 8, tx * 8), bool)
    dil[:, :H, :W] = masks[0]
    dil = dil.reshape(nb, ty, 8, tx, 8).transpose(0, 1, 3, 2, 4).reshape(nb, ty, tx, 64)[live]
    tids = tile_ids[live]
    kept = np.where(dil, -1, tids)
    colour_only = n_tile - np.array([len(set(t[t >= 0]) & set(k[k >= 0])) for t, k in zip(tids, kept)])

    def hist(x):
        return {'mean': round(float(x.mean()), 3), 'p50': int(np.percentile(x, 50)), 'p90': int(np.percentile(x, 90)),
                'p99': int(np.percentile(x, 99)), 'max': int(x.max()),
                'counts': {int(k): int(v) for k, v in zip(*np.unique(x, return_counts=True))}}

    out = {'workload': workload, 'images': int(nb), 'H': H, 'W': W, 'C': C, 'tiles': int(flagged.size),
           'flagged_share': round(float(flagged.mean()), 4), 'live_share': round(float(live.mean()), 4),
           'faces_tile_ring': hist(n_all), 'over_24': int((n_all > 24).sum()), 'over_32': int((n_all > 32).sum()),
           'faces_owning_pixels': hist(n_tile), 'faces_ring_only': hist(n_all - n_tile),
           'faces_colour_only': hist(colour_only)}
    if len(masks) == 2:
        near = np.zeros_like(ids, bool)
        c = ids >= 0
        near[:, 1:-1, 1:-1] = c[:, 1:-1, 1:-1] | c[:, :-2, 1:-1] | c[:, 2:, 1:-1] | c[:, 1:-1, :-2] | c[:, 1:-1, 2:]
        out['groups_disagree_share'] = round(float((masks[0] != masks[1])[near].mean()), 5)
        out['dilated_share'] = [round(float(m[near].mean()), 5) for m in masks]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('libs', nargs='*')
    ap.add_argument('--workloads', default='cfg3,cfg4,cfg5,cube')
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--round', type=int, default=0)
    ap.add_argument('--one', action='store_true')
    ap.add_argument('--census', action='store_true')
    ap.add_argument('--images', type=int, default=2)
    args = ap.parse_args()
    if args.census:
        for w in args.workloads.split(','):
            print(json.dumps(census(w, args.images)), flush=True)
        return
    if args.one:
        return one(args)
    libs = args.libs or [os.path.join(ROOT, 'dirt_b200', 'libdirt_b200.so')]
    for rnd in range(args.rounds):
        for lib in libs:
            env = dict(os.environ, DIRT_B200_LIB=os.path.abspath(lib))
            cmd = [sys.executable, os.path.abspath(__file__), '--one', '--workloads', args.workloads, '--steps', str(args.steps),
                   '--round', str(rnd)]
            proc = subprocess.run(cmd, env=env, capture_output=True, text=True)
            line = [l for l in proc.stdout.splitlines() if l.startswith('{')]
            print(line[-1] if line else json.dumps({'lib': os.path.basename(lib), 'round': rnd,
                                                    'error': (proc.stderr or proc.stdout)[-400:]}), flush=True)


if __name__ == '__main__':
    main()
