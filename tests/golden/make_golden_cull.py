"""Records what THE REFERENCE'S OWN cull_scan (scripts/eval_dtu/evaluate_single_scene.py:19-101) computes, for
diff_surfel_rasterization.chamfer.cull_scan (DESIGN.md §7n).

The script is loaded with runpy (not as __main__) and its cull_scan is called unmodified on data written to a
temporary directory: masks written with cv2.imwrite and read back by the reference's cv2.imread, a cameras.npz
written with np.savez, and empty files under images/ for its glob.  cv2, numpy and torch are real and run on the
CPU.  What is stubbed:
  * torch.Tensor.cuda is the identity;
  * skimage.morphology: binary_dilation is scipy.ndimage.binary_dilation with border_value 0 (what skimage calls),
    and disk returns {dx^2 + dy^2 <= r^2} for the case's radius r in place of the hard-coded 24 (the cases at r = 24
    are the reference's footprint);
  * trimesh: load serves the case's vertices (float64), faces and vertex colours; update_vertices and update_faces
    follow trimesh's documented semantics (an all-True mask returns early; otherwise faces are re-indexed through
    the inverse map, with 0 for dropped vertices, and vertices and colours are masked; update_faces masks the faces);
    export records vertices, faces and colours;
  * tqdm (the bar passes its iterable through) and imageio (unused) are no-ops.
torch.inverse, Tensor.__matmul__ and F.grid_sample are wrapped to record each view's w2c, the 4 x 4 product
intrinsic @ w2c (A), the grid and the sampled values, and the dilated mask grid_sample reads.

Writes tests/golden/ref_cull.npz.  Re-running gives the same file bit for bit.

Usage:  python tests/golden/make_golden_cull.py
"""
import glob
import io
import os
import runpy
import sys
import tempfile
import types
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPT_DIR = "/root/reference/scripts/eval_dtu"
SCRIPT = os.path.join(SCRIPT_DIR, "evaluate_single_scene.py")
IMAGE = (1600, 1200)       # the reference's hard-coded W, H


# ---- dyadic cameras: every float32 step of rule 3 is exact (checked below) ----

def dyadic_cameras(deltas, s=2.0, t=(0.25, -0.5, 0.75)):
    """world and scale matrices whose A = K [I | delta] with K = [[1599, 0, 799.5], [0, 1199, 599.5], [0, 0, 1]]:
    gx = 2 (x + dx) / (z + dz) exactly, and likewise gy."""
    K = np.array([[1599.0, 0, 799.5], [0, 1199.0, 599.5], [0, 0, 1.0]])
    S = np.eye(4)
    S[:3, :3] *= s
    S[:3, 3] = t
    world = []
    for dl in deltas:
        C = np.asarray(t) - s * np.asarray(dl, np.float64)          # A = P / s = K [I | (t - C) / s]
        Wm = np.eye(4)
        Wm[:3, :4] = K @ np.hstack([np.eye(3), -C[:, None]])
        world.append(Wm)
    return np.array(world), np.array([S] * len(deltas))


def dyadic_verts(rng, n, delta, mask_shape, inside=False):
    """Vertices for view `delta`: z + dz in {64, 128, -64}; gx, gy on half pixels of the mask, at exactly +-1, or
    on a 1/64 grid in (-1.25, 1.25).  inside: in front of the view and inside its frame."""
    Hm, Wm = mask_shape
    zc = rng.choice([64.0, 128.0, -64.0], n, p=[0.5, 0.5, 0.0] if inside else [0.45, 0.35, 0.2])
    gx = np.where(rng.random(n) < 0.4, (2 * rng.integers(0, Wm - 1, n) + 1) / (Wm - 1) - 1,
                  rng.integers(-80, 81, n) / 64.0)
    gy = np.where(rng.random(n) < 0.4, (2 * rng.integers(0, Hm - 1, n) + 1) / (Hm - 1) - 1,
                  rng.integers(-80, 81, n) / 64.0)
    if inside:
        gx, gy = np.clip(gx, -63 / 64, 63 / 64), np.clip(gy, -63 / 64, 63 / 64)
    else:
        edge = rng.random(n) < 0.1
        gx = np.where(edge, rng.choice([-1.0, 1.0], n), gx)
        edge = rng.random(n) < 0.1
        gy = np.where(edge, rng.choice([-1.0, 1.0], n), gy)
    x = gx * zc / 2 - delta[0]
    y = gy * zc / 2 - delta[1]
    return np.stack([x, y, zc - delta[2]], 1)


def blob_masks(rng, n, shape, blobs=3, noise=0.0, any_value=True):
    """Elliptic blobs and speckle; set pixels hold random nonzero values, or 255 as DTU's masks do."""
    H, W = shape
    yy, xx = np.mgrid[0:H, 0:W]
    out = []
    for _ in range(n):
        m = np.zeros(shape, bool)
        for _ in range(blobs):
            cy, cx = rng.uniform(0, H), rng.uniform(0, W)
            ry, rx = rng.uniform(0.1, 0.35) * H, rng.uniform(0.1, 0.35) * W
            m |= ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1
        m |= rng.random(shape) < noise
        out.append(np.where(m, rng.integers(1, 256, shape) if any_value else 255, 0).astype(np.uint8))
    return np.array(out)


def random_faces(rng, M, F, skip=0):
    """F faces over vertices [0, M - skip): the last `skip` vertices stay unreferenced."""
    return np.stack([rng.choice(M - skip, 3, replace=False) for _ in range(F)]).astype(np.int64)


def real_cameras(rng, n, s=300.0):
    """DTU-like cameras (K of a 1600 x 1200 DTU view, rotations looking at the origin from about 2.5 units of the
    normalised space) with a scale matrix of the DTU kind."""
    K = np.array([[2892.33, 0.0, 823.205], [0.0, 2883.18, 619.07], [0.0, 0.0, 1.0]])
    S = np.eye(4)
    S[:3, :3] *= s
    S[:3, 3] = rng.normal(size=3) * 50
    world = []
    for _ in range(n):
        c = rng.normal(size=3)
        c = c / np.linalg.norm(c) * 2.5
        f = -c / np.linalg.norm(c)
        up = np.array([0.0, 1.0, 0.0]) + 0.1 * rng.normal(size=3)
        r0 = np.cross(up, f)
        r0 /= np.linalg.norm(r0)
        r1 = np.cross(f, r0)
        R = np.stack([r0, r1, f])
        Cw = S[:3, :3] @ c + S[:3, 3]                    # the centre in world units
        Wm = np.eye(4)
        Wm[:3, :4] = (0.37 if len(world) % 2 == 0 else -0.37) * K @ np.hstack([R, -R @ Cw[:, None]])
        world.append(Wm)
    return np.array(world), np.array([S] * n)


def cases():
    rng = np.random.default_rng(20261017)
    out = []
    shape = (33, 65)                                     # Hm - 1 = 32, Wm - 1 = 64
    deltas = [(0.5, -1.0, 64.0), (1.5, 0.25, 64.0)]
    world, scale = dyadic_cameras(deltas)

    def dy(name, masks, n=600, F=700, skip=20, radius=2, colors=True, inside=False):
        v = np.concatenate([dyadic_verts(rng, n // 2, deltas[0], shape, inside),
                            dyadic_verts(rng, n - n // 2, deltas[1], shape, inside)])
        f = random_faces(rng, n, F, skip)
        c = rng.integers(0, 256, (n, 4)).astype(np.uint8) if colors else None
        out.append(dict(name=name, kind="exact", verts=v, faces=f, colors=c, masks=masks, world=world, scale=scale,
                        radius=radius))

    dy("dyadic", blob_masks(rng, 2, shape, noise=0.02))
    dy("dyadic_r1", blob_masks(rng, 2, shape, blobs=2, noise=0.05), radius=1)
    dy("all_kept", np.full((2,) + shape, 255, np.uint8))
    dy("none_kept", np.zeros((2,) + shape, np.uint8), F=300, inside=True)
    dy("empty_mask", np.stack([blob_masks(rng, 1, shape, blobs=4)[0], np.zeros(shape, np.uint8)]))
    dy("full_mask", np.stack([np.ones(shape, np.uint8), blob_masks(rng, 1, shape)[0]]))
    dy("r0", blob_masks(rng, 2, shape, noise=0.1), radius=0)
    dy("no_colors", blob_masks(rng, 2, shape), colors=False, skip=0)
    # DTU size: three 1600 x 1200 masks at disk(24), realistic cameras; and masks of another shape
    world_r, scale_r = real_cameras(rng, 3)
    n = 3000
    v = rng.normal(size=(n, 3)) * 0.35                   # the normalised space the mesh is extracted in
    f = random_faces(rng, n, 3600, skip=100)
    big = blob_masks(rng, 3, (1200, 1600), blobs=2, noise=0.0001, any_value=False)
    out.append(dict(name="dtu_size", kind="bound", verts=v, faces=f, colors=rng.integers(0, 256, (n, 3)).astype(
        np.uint8), masks=big, world=world_r, scale=scale_r, radius=24))
    out.append(dict(name="mismatch", kind="bound", verts=v[:1000], faces=random_faces(rng, 1000, 1000), colors=None,
                    masks=blob_masks(rng, 3, (300, 400), blobs=2, noise=0.001, any_value=False), world=world_r,
                    scale=scale_r,
                    radius=5))
    return out


def run_case(c, tmp):
    import cv2
    import scipy.ndimage as ndi
    import torch
    import torch.nn.functional as F
    inst = os.path.join(tmp, c["name"])
    os.makedirs(os.path.join(inst, "images"))
    os.makedirs(os.path.join(inst, "mask"))
    N = len(c["masks"])
    cams = {}
    for k in range(N):
        open(os.path.join(inst, "images", f"{k:06d}.png"), "wb").close()
        assert cv2.imwrite(os.path.join(inst, "mask", f"{k:03d}.png"), c["masks"][k])
        cams[f"world_mat_{k}"], cams[f"scale_mat_{k}"] = c["world"][k], c["scale"][k]
    np.savez(os.path.join(inst, "cameras.npz"), **cams)
    rec = {"w2c": [], "A": [], "grid": [], "sample": [], "dilated": []}

    morph = types.ModuleType("skimage.morphology")
    r = c["radius"]
    morph.disk = lambda radius: (np.arange(-r, r + 1)[:, None] ** 2 + np.arange(-r, r + 1)[None] ** 2 <= r * r
                                 ).astype(np.uint8)
    morph.binary_dilation = lambda image, footprint: ndi.binary_dilation(image, structure=footprint, border_value=0)
    sk = types.ModuleType("skimage")
    sk.morphology = morph
    tq = types.ModuleType("tqdm")
    tq.tqdm = lambda it, *a, **k: it
    io_stub = types.ModuleType("imageio")

    class Visual:
        def __init__(self, colors):
            self.vertex_colors = colors

    class Mesh:
        def __init__(self):
            self.vertices = np.array(c["verts"], np.float64)
            self.faces = np.array(c["faces"], np.int64)
            self.visual = Visual(None if c["colors"] is None else np.array(c["colors"]))

        def update_vertices(self, mask):
            mask = np.asanyarray(mask)
            if mask.dtype.name == "bool" and mask.all():
                return
            inverse = np.zeros(len(self.vertices), dtype=np.int64)
            inverse[mask] = np.arange(mask.sum())
            self.faces = inverse[self.faces.reshape(-1)].reshape((-1, 3))
            if self.visual.vertex_colors is not None:
                self.visual.vertex_colors = self.visual.vertex_colors[mask]
            self.vertices = self.vertices[mask]

        def update_faces(self, valid):
            mask = np.asanyarray(valid)
            if mask.dtype.name == "bool" and mask.all():
                return
            self.faces = self.faces[mask]

        def export(self, path):
            rec["out_verts"] = np.array(self.vertices)
            rec["out_faces"] = np.array(self.faces, np.int64)
            rec["out_colors"] = self.visual.vertex_colors

    tm = types.ModuleType("trimesh")
    tm.load = lambda path: Mesh()

    real_inverse, real_matmul, real_gs, real_cuda = torch.inverse, torch.Tensor.__matmul__, F.grid_sample, \
        torch.Tensor.cuda

    def inverse(x):
        y = real_inverse(x)
        rec["w2c"].append(y.numpy().copy())
        return y

    def matmul(a, b):
        y = real_matmul(a, b)
        if a.shape == (4, 4) and b.shape == (4, 4):
            rec["A"].append(y.numpy().copy())
        return y

    def grid_sample(inp, grid, **kw):
        y = real_gs(inp, grid, **kw)
        rec["dilated"].append(inp[0, 0].numpy() != 0)
        rec["grid"].append(grid[0, 0].numpy().copy())
        rec["sample"].append(y[0, -1, 0].numpy().copy())
        return y

    mods = ("skimage", "skimage.morphology", "trimesh", "tqdm", "imageio")
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update({"skimage": sk, "skimage.morphology": morph, "trimesh": tm, "tqdm": tq, "imageio": io_stub})
    sys.path.insert(0, SCRIPT_DIR)
    torch.inverse, torch.Tensor.__matmul__, F.grid_sample = inverse, matmul, grid_sample
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        g = runpy.run_path(SCRIPT, run_name="evaluate_single_scene")
        g["cull_scan"](1, "mesh.ply", os.path.join(tmp, "culled_mesh.ply"), inst)
    finally:
        torch.inverse, torch.Tensor.__matmul__, F.grid_sample, torch.Tensor.cuda = real_inverse, real_matmul, \
            real_gs, real_cuda
        sys.path.remove(SCRIPT_DIR)
        for k, m in saved.items():
            if m is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = m
    # the reference reads the masks back in sorted glob order: the order written
    assert sorted(glob.glob(os.path.join(inst, "mask", "*.png"))) == \
        [os.path.join(inst, "mask", f"{k:03d}.png") for k in range(N)]
    return rec


def check_exact(c, A):
    """For the dyadic cases: no float32 step of rule 3 rounds (d = c2 exactly: the 1e-6 is lost), so the decisions
    do not depend on the operation order."""
    v = c["verts"].astype(np.float32).astype(np.float64)
    assert np.array_equal(v, c["verts"])
    for k in range(len(A)):
        a = A[k].astype(np.float64)
        for row in range(3):
            acc = 0.0
            for j in range(3):
                p = a[row, j] * v[:, j]
                assert np.array_equal(p.astype(np.float32), p)
                acc = acc + p
                assert np.array_equal(acc.astype(np.float32), acc)
            acc = acc + a[row, 3]
            assert np.array_equal(acc.astype(np.float32), acc)
            if row == 2:
                c2 = acc
        d = (c2.astype(np.float32) + np.float32(1e-6)).astype(np.float64)
        assert np.array_equal(d, c2), "d is not exact"
        for row, side, ms in ((0, IMAGE[0], c["masks"].shape[2]), (1, IMAGE[1], c["masks"].shape[1])):
            cr = a[row, :3] @ v.T + a[row, 3]
            q = cr / d
            g = (q / (side - 1) - 0.5) * 2
            f = (g + 1) / 2 * (ms - 1)
            for val in (q, q / (side - 1), g, f):
                assert np.array_equal(val.astype(np.float32).astype(np.float64), val), "a step rounds"


def main():
    import torch
    torch.set_num_threads(1)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for c in cases():
            n = c["name"]
            rec = run_case(c, tmp)
            N = len(c["masks"])
            A = np.array(rec["A"])
            assert A.shape == (N, 4, 4) and len(rec["grid"]) == N
            if c["kind"] == "exact":
                check_exact(c, A[:, :3])
            out[f"{n}.kind"] = np.array(c["kind"])
            out[f"{n}.verts"] = np.asarray(c["verts"], np.float64)
            out[f"{n}.faces"] = np.asarray(c["faces"], np.int64)
            out[f"{n}.masks"] = c["masks"]
            out[f"{n}.world_mats"], out[f"{n}.scale_mats"] = c["world"], c["scale"]
            out[f"{n}.radius"] = np.array(c["radius"], np.int64)
            out[f"{n}.A"] = A
            out[f"{n}.w2c"] = np.array(rec["w2c"])
            out[f"{n}.grid"] = np.array(rec["grid"])
            out[f"{n}.sample"] = np.array(rec["sample"])
            out[f"{n}.dilated_bits"] = np.packbits(np.array(rec["dilated"]), axis=-1)
            out[f"{n}.out_verts"], out[f"{n}.out_faces"] = rec["out_verts"], rec["out_faces"]
            if c["colors"] is not None:
                out[f"{n}.colors"] = c["colors"]
                out[f"{n}.out_colors"] = rec["out_colors"]
    path = os.path.join(HERE, "ref_cull.npz")
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(out):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(out[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    print(path, os.path.getsize(path), "bytes;", sum(1 for k in out if k.endswith(".kind")), "cases")


if __name__ == "__main__":
    main()
