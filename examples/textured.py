"""Textured, lit cube through the deferred-shading entry point -- the scene of the reference's samples/textured.py
(UV-mapped cube, G-buffer of [mask, u, v, normal], texture lookup and Lambertian lighting in the shader function), with
torch in place of TensorFlow and a procedural texture in place of the photograph.

    python examples/textured.py [out.png]

`main()` shades with the package's CUDA lookup, `dirt_b200.sample_texture`.  `sample_texture` below is its restatement in
plain torch: it runs on any device (tests/test_helpers_cpu.py checks it on the CPU) and the GPU tests compare the CUDA op
with it bit for bit.  `uvs_to_pixel_indices` is the package's (plain torch as well).  Only `main()` needs the GPU.
"""
import functools
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))

from dirt_b200.texture import uvs_to_pixel_indices  # noqa: E402  (plain torch, any device)

frame_width, frame_height = 640, 480


def sample_texture(texture, indices, mode='bilinear'):
    """texture [H, W, C], fractional (row, column) indices [..., 2] -> [..., C] (samples/textured.py:30-60).  The four
    texels of a bilinear lookup wrap around the texture edge (the sample leaves that gather out of range)."""
    H, W = texture.shape[:2]
    if mode == 'nearest':
        idx = indices.long()
        return texture[idx[..., 0].clamp(0, H - 1), idx[..., 1].clamp(0, W - 1)]
    if mode != 'bilinear':
        raise NotImplementedError(mode)
    floor = indices.floor()
    frac = indices - floor
    r0, c0 = floor[..., 0].long() % H, floor[..., 1].long() % W
    r1, c1 = (r0 + 1) % H, (c0 + 1) % W
    fr, fc = frac[..., :1], frac[..., 1:]
    return (texture[r0, c0] * (1. - fc) * (1. - fr) + texture[r0, c1] * fc * (1. - fr) +
            texture[r1, c0] * (1. - fc) * fr + texture[r1, c1] * fc * fr)


def checker_texture(size=256, squares=8, device=None):
    """A coloured checkerboard [size, size, 3] in [0, 1]."""
    i = torch.arange(size, device=device)
    on = (((i[:, None] * squares) // size + (i[None, :] * squares) // size) % 2).to(torch.float32)[..., None]
    ramp = torch.stack([i[:, None].expand(size, size), i[None, :].expand(size, size), (size - 1 - i)[:, None].expand(size, size)], -1)
    return on * (0.3 + 0.7 * ramp.to(torch.float32) / (size - 1)) + (1. - on) * 0.15


def build_cube():
    """Six quads with their own vertices and uv coordinates (the uv layout of samples/textured.py:66-84)."""
    vertices, uvs, faces = [], [], []

    def add_quad(quad_vertices, quad_uvs):
        index = len(vertices)
        faces.extend([[index + 2, index + 1, index], [index, index + 3, index + 2]])
        vertices.extend(quad_vertices)
        uvs.extend(quad_uvs)

    add_quad([[-1, -1, 1], [1, -1, 1], [1, 1, 1], [-1, 1, 1]], [[0.1, 0.9], [0.9, 0.9], [0.9, 0.1], [0.1, 0.1]])         # front
    add_quad([[-1, -1, -1], [1, -1, -1], [1, 1, -1], [-1, 1, -1]], [[1, 1], [0, 1], [0, 0], [1, 0]])                     # back
    add_quad([[1, 1, 1], [1, 1, -1], [1, -1, -1], [1, -1, 1]], [[0.3, 0.25], [0.6, 0.25], [0.6, 0.55], [0.3, 0.55]])     # right
    add_quad([[-1, 1, 1], [-1, 1, -1], [-1, -1, -1], [-1, -1, 1]], [[0.4, 0.4], [0.5, 0.4], [0.5, 0.5], [0.4, 0.5]])     # left
    add_quad([[-1, 1, -1], [1, 1, -1], [1, 1, 1], [-1, 1, 1]], [[0, 0], [2, 0], [2, 2], [0, 2]])                         # top
    add_quad([[-1, -1, -1], [1, -1, -1], [1, -1, 1], [-1, -1, 1]], [[0, 0], [2, 0], [2, 2], [0, 2]])                     # bottom
    return vertices, uvs, faces


def shader_fn(gbuffer, texture, light_direction, sample=sample_texture):
    """G-buffer [H, W, 6] = (mask, u, v, nx, ny, nz) -> shaded pixels [H, W, 3] (samples/textured.py:117-143).
    `sample`: the texture lookup, the torch restatement by default, `dirt_b200.sample_texture` on the GPU."""
    from dirt_b200 import lighting
    mask, uvs, normals = gbuffer[..., :1], gbuffer[..., 1:3], gbuffer[..., 3:]
    unlit = sample(texture, uvs_to_pixel_indices(uvs, texture.shape[:2]))
    ambient = unlit * 0.4
    diffuse = lighting.diffuse_directional(normals.reshape(-1, 3), unlit.reshape(-1, 3), light_direction,
                                           light_color=torch.full((3,), 0.6, device=gbuffer.device), double_sided=True)
    diffuse = diffuse.reshape(unlit.shape)
    background = torch.tensor([0., 0., 0.3], device=gbuffer.device)
    return (diffuse + ambient) * mask + background * (1. - mask)


def main():
    import dirt_b200 as dirt
    from dirt_b200 import lighting, matrices
    device = torch.device('cuda')
    vertices, uvs, faces = build_cube()
    vertices_object = torch.tensor(vertices, dtype=torch.float32, device=device)
    uvs = torch.tensor(uvs, dtype=torch.float32, device=device)
    faces = torch.tensor(faces, dtype=torch.int32, device=device)
    texture = checker_texture(device=device).requires_grad_(True)
    light_direction = torch.tensor([1., 0., 0.], device=device, requires_grad=True)

    vertices_object = torch.cat([vertices_object, torch.ones_like(vertices_object[:, -1:])], dim=1).requires_grad_(True)
    vertices_world = vertices_object @ matrices.rodrigues([0., 0.6, 0.]).to(device)
    normals_world = lighting.vertex_normals(vertices_world, faces)
    view_matrix = matrices.compose(matrices.translation([0., -2., -3.2]), matrices.rodrigues([-0.5, 0., 0.])).to(device)
    projection_matrix = matrices.perspective_projection(near=0.1, far=20., right=0.1, aspect=float(frame_height) / frame_width).to(device)
    vertices_clip = vertices_world @ view_matrix @ projection_matrix

    # G-buffer attributes per vertex: coverage mask, uv, world-space normal
    attributes = torch.cat([torch.ones_like(uvs[:, :1]), uvs, normals_world], dim=1)
    pixels = dirt.rasterise_deferred(
        background_attributes=torch.zeros([frame_height, frame_width, 6], device=device),
        vertices=vertices_clip, vertex_attributes=attributes, faces=faces,
        shader_fn=functools.partial(shader_fn, sample=dirt.sample_texture), shader_additional_inputs=[texture, light_direction])

    loss = -pixels.mean()   # a toy loss: gradients reach the geometry, the texture and the light
    loss.backward()
    print('rendered %dx%d; |d loss / d vertices| max = %.3e, d texture touched %d texels, d light = %s'
          % (frame_width, frame_height, float(vertices_object.grad.abs().max()), int((texture.grad.abs().sum(-1) > 0).sum()),
             [round(float(x), 5) for x in light_direction.grad]))

    out = sys.argv[1] if len(sys.argv) > 1 else None
    if out:
        try:
            import cv2
            cv2.imwrite(out, (pixels.detach().clamp(0, 1) * 255).byte().cpu().numpy()[:, :, ::-1])
            print('wrote', out)
        except ImportError:
            print('cv2 not available; image not written')


if __name__ == '__main__':
    main()
