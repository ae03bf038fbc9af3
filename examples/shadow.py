"""Shadow mapping through the renderer: the deferred sample's cube over a ground plane under a directional light, and two
inverse problems that only the shadow can answer.

    python examples/shadow.py [--steps N]

The light's map comes from `lighting.shadow_map` (the cube and the floor rasterised from the light, through
`orthographic_projection` composed with a `rodrigues` rotation), and the shader of `rasterise_batch_deferred` is
ambient + `diffuse_directional` x `shadow_visibility` on a G-buffer of [mask, position, normal].  `main` fits
  (a) the light's direction, from renders of the whole scene, and
  (b) the cube's translation over the floor, from renders in which the cube is outside the camera's view, so only its
      shadow is seen,
each from a perturbed start, and prints the image losses and parameter errors before and after.
"""
import argparse
import math
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))

from examples.deferred import build_cube   # noqa: E402

SIZE = 192          # frame width and height
MAP = 512           # shadow-map width and height


def scene(device):
    """Object-space cube (half size 0.5, per-face normals) and floor (y = 0, 8 x 8) as one mesh: positions [V, 3],
    normals [V, 3], faces [F, 3], and the number of cube vertices."""
    from dirt_b200 import lighting
    v, f = build_cube()
    cube = torch.tensor(v, dtype=torch.float32, device=device) * 0.5
    faces = torch.tensor(f, dtype=torch.int32, device=device)
    cube, faces = lighting.split_vertices_by_face(cube, faces)
    cube_normals = lighting.vertex_normals_pre_split(cube, faces)
    floor = torch.tensor([[-4., 0., -4.], [4., 0., -4.], [4., 0., 4.], [-4., 0., 4.]], device=device)
    floor_faces = torch.tensor([[0, 2, 1], [0, 3, 2]], dtype=torch.int32, device=device) + cube.shape[0]
    normals = torch.cat([cube_normals, torch.tensor([[0., 1., 0.]], device=device).expand(4, 3)])
    return cube, floor, normals, torch.cat([faces, floor_faces]), cube.shape[0]


def light(angles, device):
    """The light's world -> clip matrix (a rotation by `angles`, then an orthographic box of 10 x 10 x 20 centred on
    the origin) and the direction it travels in the world."""
    from dirt_b200 import matrices
    rotation = matrices.rodrigues(angles[None])[0]
    view = rotation @ matrices.translation(torch.tensor([0., 0., -10.], device=device))
    projection = matrices.orthographic_projection(-5., 5., -5., 5., 0.1, 20.).to(device)
    return view @ projection, -rotation[:3, 2]


def camera(eye, target, device):
    """World -> clip of a camera at `eye` looking at `target` (y up), with a 40-degree square view."""
    from dirt_b200 import matrices
    forward = torch.nn.functional.normalize(torch.tensor(target) - torch.tensor(eye), dim=0)
    right = torch.nn.functional.normalize(torch.linalg.cross(forward, torch.tensor([0., 1., 0.])), dim=0)
    up = torch.linalg.cross(right, forward)
    view = torch.eye(4)
    view[:3, :3] = torch.stack([right, up, -forward], 1)
    view[3, :3] = -torch.tensor(eye) @ view[:3, :3]
    near = 0.1
    return (view @ matrices.perspective_projection(near, 50., near * math.tan(math.radians(20.)), 1.)).to(device)


def shader_fn(gbuffer, light_matrix, light_direction, shadow_map):
    """G-buffer [1, H, W, 7] = (mask, position, normal) -> pixels [1, H, W, 1]: ambient 0.2 plus Lambert under the
    light, times its visibility in the shadow map."""
    from dirt_b200 import lighting
    mask, positions, normals = gbuffer[..., :1], gbuffer[..., 1:4], gbuffer[..., 4:7]
    B, H, W, _ = gbuffer.shape
    albedo = torch.ones_like(mask)
    diffuse = lighting.diffuse_directional(normals.reshape(B, -1, 3), albedo.reshape(B, -1, 1), light_direction[None],
                                           torch.ones((B, 1), device=gbuffer.device), double_sided=False)
    vis = lighting.shadow_visibility(positions.reshape(B, -1, 3), light_matrix, shadow_map, radius=1, softness=0.02,
                                     bias=0.02)
    return mask * (0.2 + (diffuse * vis).reshape(B, H, W, 1))


def render(cube, floor, normals, faces, offset, angles, view_projection):
    """The scene with the cube moved by offset (x, z) and the light at `angles`, seen through view_projection."""
    import dirt_b200 as dirt
    from dirt_b200 import lighting
    dev = cube.device
    lift = torch.stack([offset[0], torch.tensor(0.5, device=dev), offset[1]])
    world = torch.cat([cube + lift, floor])
    light_matrix, light_direction = light(angles, dev)
    smap = lighting.shadow_map(world[None], faces, light_matrix[None], MAP, MAP)
    homogeneous = torch.cat([world, torch.ones_like(world[:, :1])], 1)
    attributes = torch.cat([torch.ones_like(world[:, :1]), world, normals], 1)
    return dirt.rasterise_batch_deferred(torch.zeros((1, SIZE, SIZE, 7), device=dev), (homogeneous @ view_projection)[None],
                                         attributes[None], faces[None], shader_fn,
                                         [light_matrix[None], light_direction, smap])


def fit(name, params, target_of, steps, lr):
    """Adam on params from their start to the image `target_of()` renders of the true values; returns the losses."""
    target = target_of(None).detach()
    opt = torch.optim.Adam(params, lr=lr)
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        loss = ((target_of(params) - target) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print('%s: image loss %.6f -> %.6f over %d steps' % (name, losses[0], losses[-1], steps))
    return losses


def main(steps=150):
    dev = torch.device('cuda')
    cube, floor, normals, faces, _ = scene(dev)
    true_offset = torch.tensor([0.3, -0.2], device=dev)
    true_angles = torch.tensor([-0.55, 0.4, 0.], device=dev)   # about 30 degrees above the horizon

    # (a) the light's direction, seen with the whole scene in view
    wide = camera([0., 4., 6.], [0., 0., 0.], dev)
    angles = torch.tensor([-0.45, 0.5, 0.], device=dev, requires_grad=True)
    fit('light direction', [angles],
        lambda p: render(cube, floor, normals, faces, true_offset, true_angles if p is None else p[0], wide), steps, 0.01)
    # a roll about the light's own axis leaves its direction, and so the images, unchanged: compare directions
    with torch.no_grad():
        cosine = torch.dot(light(angles, dev)[1], light(true_angles, dev)[1]).clamp(-1., 1.)
        start = torch.dot(light(torch.tensor([-0.45, 0.5, 0.], device=dev), dev)[1], light(true_angles, dev)[1])
    err_a = math.degrees(math.acos(float(cosine)))
    print('  light direction error %.3f degrees (%.3f at the start)' % (err_a, math.degrees(math.acos(float(start)))))

    # (b) the cube's translation, seen only through its shadow: a camera 1.5 above the floor looks down at the far part
    # of the shadow, 1.6 from the cube along the light
    _, direction = light(true_angles, dev)
    along = torch.nn.functional.normalize(direction[[0, 2]], dim=0)
    target = [float(true_offset[0] + 1.6 * along[0]), 0., float(true_offset[1] + 1.6 * along[1])]
    down = camera([target[0], 1.5, target[2] + 0.01], target, dev)
    offset = torch.tensor([0.1, 0.0], device=dev, requires_grad=True)
    with torch.no_grad():
        corners = torch.cat([cube + torch.stack([true_offset[0], torch.tensor(0.5, device=dev), true_offset[1]]),
                             torch.ones((cube.shape[0], 1), device=dev)], 1) @ down
        ndc = corners[:, :2] / corners[:, 3:]
        in_view = ((corners[:, 3] > 0) & (ndc.abs() <= 1).all(1)).any()
    print('cube corners in the camera\'s view: %s' % bool(in_view))
    fit('cube translation (shadow only)', [offset],
        lambda p: render(cube, floor, normals, faces, true_offset if p is None else p[0], true_angles, down), steps, 0.01)
    err_b = (offset - true_offset).norm().item()
    print('  cube offset %s (true %s), error %.4f' % ([round(float(x), 4) for x in offset],
                                                       [round(float(x), 4) for x in true_offset], err_b))
    return err_a, err_b


if __name__ == '__main__':
    parser = argparse.ArgumentParser()
    parser.add_argument('--steps', type=int, default=150)
    main(parser.parse_args().steps)
