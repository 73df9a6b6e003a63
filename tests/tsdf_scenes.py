"""Scenes for the TSDF field (tests/tsdf_ref.py, DESIGN.md §7i): analytic views of a sphere on a plane, and the
sample points that meet the rules' edges.

A view is a camera of surfel_scenes.make_camera on a ring around the origin, looking at it, with a (1,H,W) depth map
and a (3,H,W) RGB map.  Each pixel's depth is the view-space z of the first hit of its ray (the ray through the
pixel's align_corners=True position, so grid_sample at that pixel returns it): the unit sphere at the origin, or
the plane y = 1.  Pixels whose ray hits neither hold 0, as empty pixels of a rendered map do; a few hold NaN.
"""
import math
import types

import numpy as np
import torch

import surfel_scenes as S


def ring_camera(W, H, yaw_deg, height, dist, fovy_deg=60.0):
    C = np.array([dist * math.sin(math.radians(yaw_deg)), height, -dist * math.cos(math.radians(yaw_deg))])
    f = -C / np.linalg.norm(C)
    r = np.cross(f, [0.0, 1.0, 0.0])
    r /= np.linalg.norm(r)
    d = np.cross(f, r)
    R = np.stack([r, d, f], 1)                   # columns: view x, y, z axes in world
    t = -R.T @ C
    return S.make_camera(W, H, fovy_deg=fovy_deg, R=R, t=t)


def analytic_maps(cam, rng, n_nan=3, sphere=((0.0, 0.0, 0.0), 1.0), plane_y=1.0):
    W, H = cam["W"], cam["H"]
    wv = cam["viewmatrix"].numpy().astype(np.float64).T            # x_view = wv @ [x, 1]
    c2w = np.linalg.inv(wv)
    u = -1 + 2 * np.arange(W) / max(W - 1, 1)
    v = -1 + 2 * np.arange(H) / max(H - 1, 1)
    dv = np.stack(np.broadcast_arrays(u[None, :] * cam["tanfovx"], v[:, None] * cam["tanfovy"], np.ones((H, W))), -1)
    dw = dv @ c2w[:3, :3].T                                          # ray per unit view z
    o = c2w[:3, 3]
    cen, rad = np.asarray(sphere[0]), sphere[1]
    oc = o - cen
    a = (dw * dw).sum(-1)
    b = 2 * (dw @ oc)
    c = oc @ oc - rad * rad
    disc = b * b - 4 * a * c
    with np.errstate(invalid="ignore", divide="ignore"):
        ts = np.where(disc >= 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), np.inf)
        ts = np.where(ts > 0, ts, np.inf)
        tp = (plane_y - o[1]) / dw[..., 1]
        tp = np.where(tp > 0, tp, np.inf)
    z = np.minimum(ts, tp)
    depth = np.where(np.isfinite(z), z, 0.0).astype(np.float32)
    hit = o + np.where(np.isfinite(z), z, 0.0)[..., None] * dw
    rgb = np.where(np.isfinite(z)[None], 0.5 + 0.5 * np.sin(np.moveaxis(hit, -1, 0) * 3.0), 0.0)
    rgb = rgb.astype(np.float32)
    for _ in range(n_nan):
        depth[rng.integers(H), rng.integers(W)] = np.nan
    if H > 1 and W > 1:                          # a NaN east of pixel (0, 0): NaN there too, at weight 0
        depth[0, 1] = np.nan
    return depth[None], rgb


def analytic_views(sizes, seed, dist=3.0):
    """[(camera namespace with .full_proj_transform, depth (1,H,W), rgb (3,H,W))] as float32 CPU tensors."""
    rng = np.random.default_rng(seed)
    out = []
    for k, (W, H) in enumerate(sizes):
        cam = ring_camera(W, H, 360.0 * k / len(sizes) + 10 * rng.random(), 0.8 * rng.random() - 0.6,
                          dist * (0.9 + 0.2 * rng.random()))
        depth, rgb = analytic_maps(cam, rng, n_nan=3 if W * H >= 100 else 1)
        view = types.SimpleNamespace(full_proj_transform=cam["projmatrix"], world_view_transform=cam["viewmatrix"],
                                     image_width=W, image_height=H, camera=cam)
        out.append((view, torch.from_numpy(depth), torch.from_numpy(rgb)))
    return out


def special_points(R):
    """Contracted-space points on the rules' edges: |y| = 0, 1 and 2 exactly, the cube corners (which uncontract
    to the opposite side of the centre) and the mid-edges."""
    pts = [[0, 0, 0], [1, 0, 0], [0, -1, 0], [0, 0, 1], [0.6, 0.8, 0], [2, 0, 0], [0, 0, -2], [0, 1.2, 1.6]]
    for sx in (-1, 1):
        for sy in (-1, 1):
            for sz in (-1, 1):
                pts.append([sx * R, sy * R, sz * R])
                pts.append([sx * R, sy * R, 0])
    return np.array(pts, np.float32)


def contract(x):
    """The reference's contraction of normalized world points (mesh_utils.py:189-191), in float32."""
    x = np.asarray(x, np.float32)
    mag = np.linalg.norm(x, axis=-1, keepdims=True).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(mag < 1, x, (np.float32(2) - np.float32(1) / mag) * (x / mag)).astype(np.float32)


def sphere_surface_points(n, rng, center, radius):
    """Contracted points on the unit sphere's surface and (world) the same points."""
    d = rng.normal(size=(n, 3))
    world = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    y = contract((world - np.asarray(center, np.float32)) / np.float32(radius))
    return y, world


def frames_of(views):
    """tsdf_ref's frame list: (M, depth, rgb) numpy float32."""
    return [(v.full_proj_transform.numpy(), d.numpy()[0], c.numpy()) for v, d, c in views]
