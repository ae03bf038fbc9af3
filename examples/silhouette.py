"""Shape from silhouettes: deform a sphere into a cube through per-vertex offsets, with and without a mesh-Laplacian
smoothness term, and optionally with a normal-consistency term.

    python examples/silhouette.py [--steps N] [--weight LAMBDA] [--consistency MU]

The target's silhouettes are rendered with `rasterise_batch` from 8 cameras around it (two rings of four, above and
below the equator).  The source is `scenes.icosphere(3)` (642 vertices) plus an offset per vertex, fitted by Adam to
    silhouette MSE + lambda * mean |laplacian|^2 + mu * mean normal_consistency
with `mesh.laplacian(..., mode='uniform')` and `mesh.normal_consistency`.  `main` runs the fit twice, at
(lambda, mu) = (--weight, 0) and (0, 0), and a third time at (--weight, --consistency) when that is given.  It prints for
each: the silhouette IoU on 6 held-out views (other azimuths and elevations) before and after, the final mean
|uniform laplacian| and mean normal consistency of the mesh, and how many faces' normals turned against their starting
normals (folds).
On an H100 at the defaults (DESIGN.md §7.16) the term leaves a 5x smoother mesh with a fifth of the folds (82 of 1280
faces against 447), at about the same held-out IoU (0.908 against 0.912, from 0.652); the figures move a little from
run to run, as the rasteriser sums vertex gradients with float atomics.  DESIGN.md §7.17 records what the
normal-consistency term changes.
"""
import argparse
import math
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))

from examples.shadow import camera   # noqa: E402

SIZE = 96           # silhouette width and height
DISTANCE = 3.5      # of every camera from the origin
CONSISTENCY = 0.3   # a normal-consistency weight mu for --consistency, from the sweep of DESIGN.md §7.17


def cameras(azimuths, elevations, device):
    """World -> clip [N, 4, 4] of cameras at DISTANCE looking at the origin, one per (azimuth, elevation) in degrees."""
    out = []
    for az, el in zip(azimuths, elevations):
        a, e = math.radians(az), math.radians(el)
        eye = [DISTANCE * math.cos(e) * math.sin(a), DISTANCE * math.sin(e), DISTANCE * math.cos(e) * math.cos(a)]
        out.append(camera(eye, [0., 0., 0.], device))
    return torch.stack(out)


def silhouettes(vertices, faces, view_projections):
    """Coverage [N, SIZE, SIZE, 1] of the mesh (vertices [V, 3], faces [F, 3] int32) from each camera."""
    import dirt_b200 as dirt
    N = view_projections.shape[0]
    homogeneous = torch.cat([vertices, torch.ones_like(vertices[:, :1])], 1)
    clip = homogeneous[None] @ view_projections
    return dirt.rasterise_batch(torch.zeros((N, SIZE, SIZE, 1), device=vertices.device), clip,
                                torch.ones((N, vertices.shape[0], 1), device=vertices.device),
                                faces[None].expand(N, -1, -1).contiguous())


def iou(a, b):
    a, b = a > 0.5, b > 0.5
    return float((a & b).sum()) / max(float((a | b).sum()), 1.)


def face_normals(vertices, faces):
    p = vertices[faces.long()]
    return torch.linalg.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0], dim=-1)


def fit(weight, steps, lr=0.005, device=None, verbose=True, consistency=0.):
    """One fit at Laplacian weight `weight` and normal-consistency weight `consistency`.  Returns a dict of what `main`
    prints."""
    from dirt_b200 import mesh, scenes
    dev = device or torch.device('cuda')
    v, f = scenes.icosphere(3)
    source = torch.tensor(v, device=dev)
    faces = torch.tensor(f, dtype=torch.int32, device=dev)
    tv, tf = scenes.cube()
    target_vertices = torch.tensor(tv, device=dev) * 0.6
    target_faces = torch.tensor(tf, dtype=torch.int32, device=dev)
    train = cameras([0., 90., 180., 270., 45., 135., 225., 315.], [25.] * 4 + [-25.] * 4, dev)
    held_out = cameras([20., 110., 200., 290., 70., 250.], [0., 50., -10., -50., 70., -70.], dev)
    with torch.no_grad():
        target = silhouettes(target_vertices, target_faces, train)
        target_held = silhouettes(target_vertices, target_faces, held_out)
        start_iou = iou(silhouettes(source, faces, held_out), target_held)
    offsets = torch.zeros_like(source, requires_grad=True)
    opt = torch.optim.Adam([offsets], lr=lr)
    for step in range(steps):
        opt.zero_grad()
        vertices = source + offsets
        data = ((silhouettes(vertices, faces, train) - target) ** 2).mean()
        smooth = mesh.laplacian(vertices, faces, 'uniform').square().sum(-1).mean()
        loss = data + weight * smooth
        if consistency:
            loss = loss + consistency * mesh.normal_consistency(vertices, faces).mean()
        loss.backward()
        opt.step()
        if verbose and (step == 0 or (step + 1) % max(steps // 4, 1) == 0):
            print('  lambda %g step %4d: silhouette MSE %.5f, mean |L|^2 %.3e' % (weight, step + 1, data.item(),
                                                                                  smooth.item()))
    with torch.no_grad():
        vertices = source + offsets
        end_iou = iou(silhouettes(vertices, faces, held_out), target_held)
        mean_l = mesh.laplacian(vertices, faces, 'uniform').norm(dim=-1).mean().item()
        start_l = mesh.laplacian(source, faces, 'uniform').norm(dim=-1).mean().item()
        mean_c = mesh.normal_consistency(vertices, faces).mean().item()
        start_c = mesh.normal_consistency(source, faces).mean().item()
        flipped = int(((face_normals(vertices, faces) * face_normals(source, faces)).sum(-1) < 0).sum())
    return {'weight': weight, 'consistency': consistency, 'held_out_iou_start': start_iou, 'held_out_iou_end': end_iou,
            'mean_laplacian_start': start_l, 'mean_laplacian_end': mean_l, 'mean_consistency_start': start_c,
            'mean_consistency_end': mean_c, 'flipped_faces': flipped, 'faces': int(faces.shape[0])}


def main(steps=300, weight=10., consistency=None):
    results = []
    runs = [(weight, 0.), (0., 0.)] + ([(weight, consistency)] if consistency is not None else [])
    for w, mu in runs:
        r = fit(w, steps, consistency=mu)
        print('lambda %g, mu %g: held-out IoU %.4f -> %.4f, mean |uniform laplacian| %.5f (sphere %.5f), mean normal '
              'consistency %.5f (sphere %.5f), faces flipped %d of %d'
              % (w, mu, r['held_out_iou_start'], r['held_out_iou_end'], r['mean_laplacian_end'],
                 r['mean_laplacian_start'], r['mean_consistency_end'], r['mean_consistency_start'], r['flipped_faces'],
                 r['faces']))
        results.append(r)
    return results


if __name__ == '__main__':
    parser = argparse.ArgumentParser()
    parser.add_argument('--steps', type=int, default=300)
    parser.add_argument('--weight', type=float, default=10.)
    parser.add_argument('--consistency', type=float, default=None, metavar='MU')
    args = parser.parse_args()
    main(args.steps, args.weight, args.consistency)
