"""Records what THE REFERENCE'S OWN post_process_mesh (utils/mesh_utils.py:22-43 of the reference) returns, for
diff_surfel_rasterization.meshpost.post_process_mesh (DESIGN.md §7k).

The reference's function runs unmodified on the CPU (make_golden.cpu_patches / stub_modules).  open3d is a stub whose
geometry.TriangleMesh is restatement (a) of tests/meshpost_ref.py (Open3D's cluster_connected_triangles,
remove_triangles_by_mask, remove_unreferenced_vertices and remove_degenerate_triangles as recalled), and whose
utility has VerbosityContextManager and VerbosityLevel; so the reference's deep copy, sort, negative indexing,
max(., 50) and mask run as written.  Per (mesh, k) it records the mask passed to remove_triangles_by_mask and the
returned vertices, triangles and vertex colours, or the type of the exception raised.

Meshes: marching cubes of the TSDF golden scene (tests/golden/ref_tsdf.npz, the restatement of tests/mcubes_ref.py at
two crops of 17^3 points) with its colours; bipyramids ("spheres") and fans of sizes above, at and below 50 faces,
with ties at the k-th count, faces interleaved; a bow-tie; duplicate faces, opposite windings and a non-manifold edge;
degenerate (a,a,b) and (a,a,a) faces and a vertex referenced only by degenerate faces; unreferenced vertices and NaN
positions; one face; no faces.  k in {1, 2, 50, 1000, 0, -1, C, C + 1}, C the mesh's number of clusters.

Writes tests/golden/ref_meshpost.npz.

Usage:  python tests/golden/make_golden_meshpost.py
"""
import contextlib
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_tsdf as MGT  # noqa: E402  (sets the paths)

REF = MGT.REF
F32 = np.float32


def tsdf_mesh():
    import mcubes_ref as MR
    import tsdf_ref as TR
    g = np.load(os.path.join(HERE, "ref_tsdf.npz"))
    frames = [(g[f"proj{f}"], g[f"depth{f}"][0], g[f"rgb{f}"]) for f in range(int(g["n_frames"]))]
    center, radius, trunc = g["center"], float(g["radius"]), 5 * float(g["voxel_size"])
    n, side, R = 2, 17, 1.2

    def values(ijk, axes):
        X, Y, Z = np.meshgrid(*axes, indexing="ij")
        pts = np.stack([X.ravel(), Y.ravel(), Z.ravel()], 1).astype(F32)
        return TR.emulate(pts, frames, center, radius, trunc)
    verts, faces, _, _ = MR.mesh(n, side, MR.crop_bounds(R, n), values, center, radius)
    colors = TR.emulate(verts, frames, center, radius, trunc, colour=True)
    return verts, faces, colors


def synthetic_meshes(rng):
    import meshpost_ref as MP
    out = {}
    # spheres and fans above, at and below 50 faces; 52 twice and 50 twice (ties), faces interleaved
    parts, v0 = [], 0
    for kind, n in (("b", 26), ("b", 25), ("f", 49), ("b", 26), ("b", 60), ("f", 50), ("b", 24), ("f", 10),
                    ("b", 3), ("f", 51)):
        f = MP.bipyramid(n, v0) if kind == "b" else MP.fan(n, v0)
        parts.append(f)
        v0 = int(f.max()) + 1
    faces = np.concatenate(parts)
    faces = faces[rng.permutation(len(faces))]
    out["spheres"] = (rng.normal(size=(v0, 3)).astype(F32), faces, rng.uniform(size=(v0, 3)).astype(F32))
    # a big grid (so that something survives the floor of 50) beside each feature
    g = MP.grid(8, 8)                                          # 98 faces over vertices 0..63
    # bow-ties: two fans of 60 faces around vertex 64 sharing only it, and two faces sharing only vertex 190
    fan_a, fan_b = MP.fan(60, 64), MP.fan(60, 125)
    fan_b[:, 0] = 64
    bow = np.array([[190, 191, 192], [190, 193, 194]])
    out["bowtie"] = (rng.normal(size=(200, 3)).astype(F32), np.concatenate([g, fan_a, bow, fan_b]), None)
    # duplicates, opposite windings, a non-manifold edge shared by 4 faces
    dup = np.array([[0, 1, 8], [0, 1, 8], [1, 0, 8], [8, 1, 0], [100, 101, 102], [100, 101, 103], [101, 100, 104],
                    [100, 101, 105], [102, 103, 106]])
    out["duplicates"] = (rng.normal(size=(110, 3)).astype(F32), np.concatenate([dup[:4], g, dup[4:]]), None)
    # degenerate faces: (a,a,b) on a grid edge, (a,a,c) through (a,a), (a,a,a); vertex 70 only in degenerate faces;
    # (80,80,81)+(80,80,82) form their own cluster
    deg = np.array([[9, 9, 10], [9, 9, 70], [11, 11, 11], [70, 70, 9], [80, 80, 81], [80, 80, 82], [83, 83, 83]])
    out["degenerate"] = (rng.normal(size=(90, 3)).astype(F32), np.concatenate([g[:50], deg, g[50:]]),
                         rng.uniform(size=(90, 4)).astype(F32))
    # unreferenced input vertices and NaN positions
    M = 150
    remap = np.sort(rng.choice(M, 64, replace=False))
    v = rng.normal(size=(M, 3)).astype(F32)
    v[remap[[3, 17, 40]], 1] = np.nan
    v[[i for i in range(M) if i not in set(remap)][:4]] = np.nan
    out["unreferenced_nan"] = (v, remap[g], rng.uniform(size=(M, 3)).astype(F32))
    out["one_face"] = (rng.normal(size=(3, 3)).astype(F32), np.array([[0, 1, 2]]), None)
    out["no_faces"] = (rng.normal(size=(5, 3)).astype(F32), np.zeros((0, 3), np.int64), None)
    return out


def main():
    import meshpost_ref as MP
    rng = np.random.default_rng(5)
    meshes = {"tsdf_mc": tsdf_mesh()}
    meshes.update(synthetic_meshes(rng))

    import make_golden as MG
    MG.cpu_patches()
    MG.stub_modules({})
    for name in ("open3d", "trimesh", "skimage", "skimage.measure", "mediapy"):
        sys.modules[name] = types.ModuleType(name)
    o3d = sys.modules["open3d"]
    o3d.geometry = types.SimpleNamespace(TriangleMesh=MP.TriangleMesh)
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a),
                                        VerbosityLevel=types.SimpleNamespace(Debug=3),
                                        VerbosityContextManager=lambda level: contextlib.nullcontext())
    mpl = sys.modules.get("matplotlib")
    if mpl is not None and not hasattr(mpl, "cm"):
        mpl.cm = types.ModuleType("matplotlib.cm")
    sys.path.insert(0, REF)
    from utils.mesh_utils import post_process_mesh

    out = {}
    for name, (v, f, c) in meshes.items():
        f = np.asarray(f, np.int64).reshape(-1, 3)
        out[f"{name}.verts"], out[f"{name}.faces"] = np.asarray(v, F32), f
        if c is not None:
            out[f"{name}.colors"] = np.asarray(c, F32)
        C = len(MP.clusters_literal(f)[1])
        ks = [1, 2, 50, 1000, 0, -1, C, C + 1]
        out[f"{name}.ks"] = np.array(ks, np.int64)
        for k in ks:
            mesh = MP.TriangleMesh(v, f, c)
            tag = f"{name}.k{k}"
            try:
                res = post_process_mesh(mesh, cluster_to_keep=k)
            except Exception as ex:                  # noqa: BLE001  (recorded: the device path must raise the same)
                out[f"{tag}.error"] = np.array(type(ex).__name__)
                continue
            assert len(mesh.masks) == 0 and len(res.masks) == 1        # the input was left alone
            out[f"{tag}.mask"] = res.masks[0]
            out[f"{tag}.verts"] = res.vertices.astype(F32)
            out[f"{tag}.faces"] = res.triangles.astype(np.int64)
            if c is not None:
                out[f"{tag}.colors"] = res.vertex_colors.astype(F32)
        print(f"{name}: {len(v)} vertices, {len(f)} faces, {C} clusters")
    np.savez_compressed(os.path.join(HERE, "ref_meshpost.npz"), **out)
    print(f"wrote ref_meshpost.npz ({os.path.getsize(os.path.join(HERE, 'ref_meshpost.npz'))} bytes)")


if __name__ == "__main__":
    main()
