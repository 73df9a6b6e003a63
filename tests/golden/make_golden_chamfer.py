"""Records what THE REFERENCE'S OWN scripts/eval_dtu/eval.py computes, for diff_surfel_rasterization.chamfer
(DESIGN.md §7m).

eval.py runs unmodified as __main__ through runpy, with real numpy, sklearn, scipy.io.loadmat (on .mat files written
here with savemat) and multiprocessing.Pool.  Only three things are stubbed:
  * open3d I/O: read_triangle_mesh / read_point_cloud serve the case's mesh, cloud or STL; write_point_cloud
    captures the two visualisation clouds and their colours;
  * tqdm (a no-op bar);
  * np.random.default_rng: every call returns a real Generator, except that shuffle(x, axis=0) of the (N,3) cloud
    records x, then applies real_rng(seed).permutation(N) to the rows.
sklearn.neighbors.NearestNeighbors is replaced by a subclass that records what radius_neighbors and kneighbors
return.  Per case it records the pre-shuffle cloud, the permutation, each row's sorted radius-neighbour indices
(as CSR), both kneighbors results, both written clouds with their colours and results.json, or the type of the
exception raised.

Writes tests/golden/ref_chamfer.npz.  Re-running gives the same file bit for bit.

Usage:  python tests/golden/make_golden_chamfer.py
"""
import io
import json
import os
import runpy
import sys
import tempfile
import types
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
EVAL = "/root/reference/scripts/eval_dtu/eval.py"
SCAN = 1


def height_mesh(nx, ny, size, rng, amp=1.0, noise=0.0):
    xs, ys = np.linspace(0, size, nx), np.linspace(0, size, ny)
    X, Y = np.meshgrid(xs, ys, indexing="ij")
    Z = amp * np.sin(X / 3.0) * np.cos(Y / 4.0) + noise * rng.standard_normal(X.shape)
    verts = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1)
    idx = np.arange(nx * ny).reshape(nx, ny)
    a, b, c, d = idx[:-1, :-1].ravel(), idx[1:, :-1].ravel(), idx[:-1, 1:].ravel(), idx[1:, 1:].ravel()
    faces = np.concatenate([np.stack([a, b, c], 1), np.stack([b, d, c], 1)])
    return verts, faces


def cases():
    rng = np.random.default_rng(20261017)
    out = []
    # bumpy height field, noisy STL (part of it > max_dist away), random ObsMask, a plane that cuts the STL
    v, f = height_mesh(24, 20, 12.0, rng, amp=1.5, noise=0.05)
    stl = np.concatenate([v[rng.integers(0, len(v), 3000)] + 0.3 * rng.standard_normal((3000, 3)),
                          rng.uniform(0, 12, (100, 3)) + [0, 0, 30.0]])
    bb = np.array([[-0.3, -0.3, -3.1], [12.3, 12.3, 3.1]])
    obs = rng.random((13, 13, 7)) < 0.8
    out.append(dict(name="bumpy", mode="mesh", verts=v, faces=f, stl=stl, obs=obs, bb=bb, res=1.0,
                    plane=np.array([0.05, -0.02, 1.0, 0.2]), seed=1, args={}))
    # dyadic cloud (pcd mode): spacing 0.25 with threshold 0.25, so most neighbour pairs lie exactly at r
    g = np.stack(np.meshgrid(np.arange(12), np.arange(10), np.arange(3), indexing="ij"), -1).reshape(-1, 3) * 0.25
    g = np.concatenate([g, g[rng.integers(0, len(g), 60)] + rng.integers(-4, 5, (60, 3)) / 64.0])
    out.append(dict(name="dyadic_pcd", mode="pcd", pcd=g, stl=g[::3] + 0.125, obs=np.ones((4, 4, 2), bool),
                    bb=np.array([[0.0, 0.0, 0.0], [3.0, 3.0, 1.0]]), res=1.0, plane=np.array([0.0, 0.0, 1.0, 0.1]),
                    seed=2, args={"--downsample_density": "0.25"}))
    # dyadic mesh vertices at threshold 0.25
    v, f = height_mesh(9, 9, 2.0, rng, amp=0.0)
    out.append(dict(name="dyadic_mesh", mode="mesh", verts=v, faces=f, stl=v + [0.0, 0.0, 0.25],
                    obs=np.ones((3, 3, 2), bool), bb=np.array([[0.0, 0.0, -0.5], [2.0, 2.0, 0.5]]), res=1.0,
                    plane=np.array([0.0, 0.0, 1.0, 0.0]), seed=3, args={"--downsample_density": "0.25"}))
    # duplicate vertices (same coordinates, other indices) and duplicate faces
    v, f = height_mesh(10, 10, 3.0, rng, amp=0.5)
    v2 = np.concatenate([v, v[:40]])
    f2 = np.concatenate([f, f[:30], f[:20] % 40 + len(v)])
    out.append(dict(name="duplicates", mode="mesh", verts=v2, faces=f2, stl=v + 0.1, obs=np.ones((4, 4, 3), bool),
                    bb=np.array([[0.0, 0.0, -1.0], [3.0, 3.0, 1.0]]), res=1.0, plane=np.array([0, 0, 1.0, 5.0]),
                    seed=4, args={}))
    # zero-area (collinear, repeated index), needle and n = 0 triangles beside ordinary ones
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [0, 1, 0], [0.05, 0.05, 0], [0.1, 0, 0], [5, 0.01, 0],
                  [0, 0, 1], [3, 3, 0], [3, 4, 0], [4, 3, 0], [0.01, 0.0, 0.0], [0.0, 0.01, 0.0]], np.float64)
    f = np.array([[0, 1, 2], [0, 0, 3], [0, 1, 3], [0, 6, 5], [0, 4, 5], [1, 3, 7], [8, 9, 10], [0, 11, 12],
                  [3, 3, 3], [0, 2, 6]])
    out.append(dict(name="degenerate", mode="mesh", verts=v, faces=f, stl=v[[0, 3, 7, 8, 9]] + 0.05,
                    obs=np.ones((6, 6, 2), bool), bb=np.array([[-0.5, -0.5, -0.5], [5.5, 5.5, 1.5]]), res=1.0,
                    plane=np.array([0.0, 0.0, 1.0, 1.0]), seed=5, args={}))
    # points on the float32 box bounds and on .5 grid rounding (patch 0.5, res 0.5, bb not representable)
    bb = np.array([[0.1, 0.2, 0.3], [2.1, 2.2, 2.3]])
    lo = (bb.astype(np.float32)[:1] - 0.5)[0].astype(np.float64)
    hi = (bb.astype(np.float32)[1:] + 0.5 * 2)[0].astype(np.float64)
    b0 = bb.astype(np.float32)[0].astype(np.float64)
    pts = [lo, hi, [lo[0], 1.0, 1.0], [hi[0], 1.0, 1.0], [1.0, np.nextafter(hi[1], -np.inf), 1.0],
           [np.nextafter(lo[0], -np.inf), 1.0, 1.0]]
    pts += [b0 + 0.5 * np.array([k + 0.5, 1.5, 2.5]) for k in range(-1, 6)]
    pts += [b0 + 0.5 * np.array([2.5, k + 0.5, 0.5]) for k in range(-1, 6)]
    out.append(dict(name="bounds_pcd", mode="pcd", pcd=np.array(pts), stl=np.array(pts) + 0.01,
                    obs=(np.arange(5 * 5 * 5).reshape(5, 5, 5) % 3) != 0, bb=bb, res=0.5,
                    plane=np.array([0.0, 0.0, 1.0, 0.0]), seed=6,
                    args={"--patch_size": "0.5", "--downsample_density": "0.01"}))
    # STL points at exactly max_dist (20) from the data and on the plane (z = 1 exactly)
    d = np.array([[0, 0, 1], [1, 0, 1], [0, 1, 1], [2, 2, 2]], np.float64)
    s = np.array([[20, 0, 1], [0, 21, 1], [1, 0, 1.5], [3, 4, 1], [0, 0, 2], [0, -20, 1], [2, 2, 22.0]])
    out.append(dict(name="maxdist_plane_pcd", mode="pcd", pcd=d, stl=s, obs=np.ones((3, 3, 3), bool),
                    bb=np.array([[0.0, 0.0, 0.0], [2.0, 2.0, 2.0]]), res=1.0, plane=np.array([0.0, 0.0, 1.0, -1.0]),
                    seed=7, args={}))
    # non-default density, patch, max_dist; visualize_threshold below and above max_dist
    v, f = height_mesh(16, 16, 8.0, rng, amp=1.0, noise=0.1)
    stl = v[rng.integers(0, len(v), 1500)] + 0.8 * rng.standard_normal((1500, 3))
    for k, vis in (("vis_below", "1.0"), ("vis_above", "8.0")):
        out.append(dict(name=f"params_{k}", mode="mesh", verts=v, faces=f, stl=stl, obs=rng.random((9, 9, 5)) < 0.7,
                        bb=np.array([[0.0, 0.0, -2.0], [8.0, 8.0, 2.0]]), res=1.0,
                        plane=np.array([0.0, 0.1, 1.0, 0.5]), seed=8,
                        args={"--downsample_density": "0.5", "--patch_size": "1.5", "--max_dist": "3.0",
                              "--visualize_threshold": vis}))
    # raising cases
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [0, 1, 0]], np.float64)
    one = np.ones((3, 3, 3), bool)
    base = dict(stl=v + 0.1, obs=one, bb=np.array([[0.0, 0, -1], [2, 2, 1]]), res=1.0,
                plane=np.array([0.0, 0, 1, 0]), seed=9)
    out.append(dict(base, name="raise_no_area", mode="mesh", verts=v, faces=np.array([[0, 1, 2], [3, 3, 0]]),
                    args={}))
    out.append(dict(base, name="raise_empty_in", mode="mesh", verts=v + [50.0, 0, 0], faces=np.array([[0, 1, 3]]),
                    args={"--patch_size": "1"}))
    out.append(dict(base, name="raise_empty_obs", mode="mesh", verts=v, faces=np.array([[0, 1, 3]]),
                    obs=np.zeros((3, 3, 3), bool), args={}))
    out.append(dict(base, name="raise_empty_above", mode="mesh", verts=v, faces=np.array([[0, 1, 3]]),
                    plane=np.array([0.0, 0, 1, -5]), args={}))
    return out


def run_case(c, tmp):
    import multiprocessing as mp
    import scipy.io
    import sklearn.neighbors as skln
    rec = {"knn": []}
    os.makedirs(os.path.join(tmp, "ObsMask"), exist_ok=True)
    scipy.io.savemat(os.path.join(tmp, "ObsMask", f"ObsMask{SCAN}_10.mat"),
                     {"ObsMask": c["obs"], "BB": c["bb"], "Res": np.array([[c["res"]]])})
    scipy.io.savemat(os.path.join(tmp, "ObsMask", f"Plane{SCAN}.mat"), {"P": c["plane"].reshape(1, 4)})

    o3d = types.ModuleType("open3d")
    o3d.io = types.SimpleNamespace()
    o3d.geometry = types.SimpleNamespace(PointCloud=lambda: types.SimpleNamespace(points=None, colors=None))
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.array(a, np.float64, copy=True))
    o3d.io.read_triangle_mesh = lambda path: types.SimpleNamespace(vertices=np.array(c["verts"], np.float64),
                                                                   triangles=np.array(c["faces"], np.int32))
    o3d.io.read_point_cloud = lambda path: types.SimpleNamespace(
        points=np.array(c["stl"] if "stl" in os.path.basename(path) else c["pcd"], np.float64))

    def write_point_cloud(path, pcd):
        rec[os.path.basename(path)] = (np.asarray(pcd.points), np.asarray(pcd.colors))
        return True
    o3d.io.write_point_cloud = write_point_cloud
    tq = types.ModuleType("tqdm")

    class Bar:
        def __init__(self, *a, **k):
            pass

        def __getattr__(self, name):
            return lambda *a, **k: None
    tq.tqdm = Bar

    real_default_rng = np.random.default_rng

    class Rng:
        def __init__(self, *a, **k):
            self._g = real_default_rng(*a, **k)

        def __getattr__(self, name):
            return getattr(self._g, name)

        def shuffle(self, x, axis=0):
            if axis == 0 and getattr(x, "ndim", 0) == 2 and x.shape[1] == 3:
                rec["pcd"] = x.copy()
                perm = real_default_rng(c["seed"]).permutation(len(x))
                rec["perm"] = perm
                x[...] = x[perm]
                return None
            return self._g.shuffle(x, axis=axis)

    class RecNN(skln.NearestNeighbors):
        def radius_neighbors(self, X=None, radius=None, return_distance=True, sort_results=False):
            out = super().radius_neighbors(X, radius=radius, return_distance=return_distance,
                                           sort_results=sort_results)
            rec["rnn"] = out
            return out

        def kneighbors(self, X=None, n_neighbors=None, return_distance=True):
            out = super().kneighbors(X, n_neighbors=n_neighbors, return_distance=return_distance)
            rec["knn"].append(out)
            return out

    saved = {k: sys.modules.get(k) for k in ("open3d", "tqdm")}
    saved_nn, saved_argv = skln.NearestNeighbors, sys.argv
    sys.modules["open3d"], sys.modules["tqdm"] = o3d, tq
    np.random.default_rng = Rng
    skln.NearestNeighbors = RecNN
    sys.argv = ["eval.py", "--data", "data.ply", "--scan", str(SCAN), "--mode", c["mode"], "--dataset_dir", tmp,
                "--vis_out_dir", tmp] + [x for kv in c["args"].items() for x in kv]
    mp.set_start_method("fork", force=True)
    try:
        runpy.run_path(EVAL, run_name="__main__")
        rec["error"] = ""
    except Exception as ex:   # noqa: BLE001  (the type is what is recorded)
        rec["error"] = type(ex).__name__
    finally:
        np.random.default_rng = real_default_rng
        skln.NearestNeighbors = saved_nn
        sys.argv = saved_argv
        for k, m in saved.items():
            if m is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = m
    res_path = os.path.join(tmp, "results.json")
    if not rec["error"]:
        with open(res_path) as fp:
            rec["results"] = json.load(fp)
        os.remove(res_path)
    return rec


def main():
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for c in cases():
            n = c["name"]
            rec = run_case(c, tmp)
            out[f"{n}.mode"] = np.array(c["mode"])
            for k in ("stl", "obs", "bb", "plane"):
                out[f"{n}.{k}"] = np.asarray(c[k])
            out[f"{n}.res"] = np.array(c["res"], np.float64)
            if c["mode"] == "mesh":
                out[f"{n}.verts"] = np.asarray(c["verts"], np.float64)
                out[f"{n}.faces"] = np.asarray(c["faces"], np.int64)
            else:
                out[f"{n}.pcd_in"] = np.asarray(c["pcd"], np.float64)
            args = {"--downsample_density": 0.2, "--patch_size": 60.0, "--max_dist": 20.0,
                    "--visualize_threshold": 10.0}
            args.update({k: float(v) for k, v in c["args"].items()})
            out[f"{n}.args"] = np.array([args["--downsample_density"], args["--patch_size"], args["--max_dist"],
                                         args["--visualize_threshold"]])
            out[f"{n}.error"] = np.array(rec["error"])
            if "pcd" in rec:
                out[f"{n}.pcd"] = rec["pcd"]
                out[f"{n}.perm"] = rec["perm"]
            if "rnn" in rec:
                rows = [np.sort(r) for r in rec["rnn"]]
                out[f"{n}.rnn_ptr"] = np.cumsum([0] + [len(r) for r in rows]).astype(np.int64)
                out[f"{n}.rnn_idx"] = np.concatenate(rows).astype(np.int64)
            for k, (dist, idx) in enumerate(rec["knn"]):
                out[f"{n}.knn{k}_dist"], out[f"{n}.knn{k}_idx"] = dist[:, 0], idx[:, 0].astype(np.int64)
            if not rec["error"]:
                out[f"{n}.d2s_points"], out[f"{n}.d2s_colors"] = rec[f"vis_{SCAN:03}_d2s.ply"]
                out[f"{n}.s2d_points"], out[f"{n}.s2d_colors"] = rec[f"vis_{SCAN:03}_s2d.ply"]
                r = rec["results"]
                out[f"{n}.results"] = np.array([r["mean_d2s"], r["mean_s2d"], r["overall"]])
    # a fixed zip (no timestamps) so that a re-run gives the same bytes
    path = os.path.join(HERE, "ref_chamfer.npz")
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(out):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(out[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    print(path, os.path.getsize(path), "bytes;", sum(1 for k in out if k.endswith(".mode")), "cases")


if __name__ == "__main__":
    main()
