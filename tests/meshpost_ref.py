"""Two independent NumPy restatements of the reference's post_process_mesh (utils/mesh_utils.py:22-43) for
diff_surfel_rasterization.meshpost (csrc/meshpost.cu, DESIGN.md §7k).  The device output must equal them exactly.

(a) literal: an edge-to-faces map and a BFS from the lowest unlabelled face give Open3D's cluster_connected_triangles
    (as recalled, unverified against Open3D: faces are adjacent when they share an unordered vertex-index pair as an
    edge, degenerate pairs included; ids in discovery order), then the reference's steps one face and one vertex at a
    time.  `TriangleMesh` wraps it in the Open3D methods post_process_mesh calls, so the reference's own function runs
    on it (tests/golden/make_golden_meshpost.py).
(b) vectorised: np.unique on edge keys, scipy's connected_components on the face-edge graph, ids canonicalised to
    the rank of each component's smallest face, bincount and searchsorted compaction.  Fast enough for meshes of
    millions of faces.
"""
import numpy as np

MIN_CLUSTER = 50


# ---- (a) literal ----------------------------------------------------------------------------------------------------

def _edges(face):
    a, b, c = (int(x) for x in face)
    return [(min(u, v), max(u, v)) for u, v in ((a, b), (b, c), (c, a))]


def clusters_literal(faces):
    """(per-face cluster id, per-cluster face count) as cluster_connected_triangles returns them."""
    faces = np.asarray(faces).reshape(-1, 3)
    edge_faces = {}
    for t, face in enumerate(faces):
        for e in _edges(face):
            edge_faces.setdefault(e, []).append(t)
    ids = np.full(len(faces), -1, np.int64)
    counts = []
    for t in range(len(faces)):
        if ids[t] >= 0:
            continue
        c = len(counts)
        ids[t] = c
        queue, n = [t], 0
        while queue:
            u = queue.pop()
            n += 1
            for e in _edges(faces[u]):
                for w in edge_faces[e]:
                    if ids[w] < 0:
                        ids[w] = c
                        queue.append(w)
        counts.append(n)
    return ids, np.asarray(counts, np.int64)


class TriangleMesh:
    """The part of open3d.geometry.TriangleMesh that post_process_mesh uses, on restatement (a).  `masks` records
    what remove_triangles_by_mask is given."""

    def __init__(self, vertices, triangles, vertex_colors=None):
        self.vertices = np.asarray(vertices, np.float64).reshape(-1, 3)
        self.triangles = np.asarray(triangles, np.int64).reshape(-1, 3)
        self.vertex_colors = None if vertex_colors is None else np.asarray(vertex_colors, np.float64)
        self.masks = []

    def cluster_connected_triangles(self):
        ids, counts = clusters_literal(self.triangles)
        return ids, counts, np.zeros(len(counts))          # areas: post_process_mesh never reads them

    def remove_triangles_by_mask(self, mask):
        mask = np.asarray(mask, bool)
        self.masks.append(mask.copy())
        self.triangles = np.asarray([t for t, m in zip(self.triangles, mask) if not m], np.int64).reshape(-1, 3)

    def remove_unreferenced_vertices(self):
        used = [False] * len(self.vertices)
        for t in self.triangles:
            for v in t:
                used[v] = True
        new, keep = {}, []
        for v, u in enumerate(used):
            if u:
                new[v] = len(keep)
                keep.append(v)
        keep = np.asarray(keep, np.int64)
        self.vertices = self.vertices[keep]
        if self.vertex_colors is not None:
            self.vertex_colors = self.vertex_colors[keep]
        self.triangles = np.asarray([[new[v] for v in t] for t in self.triangles], np.int64).reshape(-1, 3)

    def remove_degenerate_triangles(self):
        self.triangles = np.asarray([t for t in self.triangles if len({int(v) for v in t}) == 3],
                                    np.int64).reshape(-1, 3)


def post_process_literal(verts, faces, colors, k):
    """Steps 1-6 on restatement (a): (mask of removed faces, verts, faces, colors or None)."""
    m = TriangleMesh(verts, faces, colors)
    ids, counts, _ = m.cluster_connected_triangles()
    n = np.sort(counts.copy())[-k]
    n = max(n, MIN_CLUSTER)
    m.remove_triangles_by_mask(counts[ids] < n)
    m.remove_unreferenced_vertices()
    m.remove_degenerate_triangles()
    return m.masks[0], m.vertices, m.triangles, m.vertex_colors


# ---- (b) vectorised -------------------------------------------------------------------------------------------------

def clusters_vectorised(faces, n_verts):
    """(per-face cluster id, per-cluster face count) from np.unique and scipy's connected components."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    F = len(f)
    if F == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    a = f[:, [0, 1, 2]].ravel()
    b = f[:, [1, 2, 0]].ravel()
    keys = np.minimum(a, b) * np.int64(max(n_verts, 1)) + np.maximum(a, b)
    _, edge = np.unique(keys, return_inverse=True)
    E = int(edge.max()) + 1
    face = np.repeat(np.arange(F, dtype=np.int64), 3)
    g = coo_matrix((np.ones(3 * F, np.int8), (face, F + edge.ravel())), shape=(F + E, F + E))
    _, label = connected_components(g, directed=False)
    label = label[:F]
    _, first = np.unique(label, return_index=True)        # each component's smallest face
    order = np.argsort(first, kind="stable")
    rank = np.empty(len(first), np.int64)
    rank[order] = np.arange(len(first))
    comp = np.unique(label, return_inverse=True)[1].ravel()
    ids = rank[comp]
    return ids, np.bincount(ids, minlength=len(first)).astype(np.int64)


def post_process_vectorised(verts, faces, colors, k, clusters=None):
    """Steps 1-6 vectorised: (mask of removed faces, verts, faces, colors or None).  `clusters`: (ids, counts) when
    already known."""
    verts = np.asarray(verts)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    ids, counts = clusters if clusters is not None else clusters_vectorised(f, len(verts))
    n = max(np.sort(counts)[-k], MIN_CLUSTER)
    removed = counts[ids] < n
    kept = f[~removed]
    vert_map = np.flatnonzero(np.bincount(kept.ravel(), minlength=len(verts)))
    out = np.searchsorted(vert_map, kept).reshape(-1, 3)
    nondeg = (out[:, 0] != out[:, 1]) & (out[:, 1] != out[:, 2]) & (out[:, 0] != out[:, 2])
    return (removed, verts[vert_map], out[nondeg].astype(np.int64),
            None if colors is None else np.asarray(colors)[vert_map])


# ---- meshes ----------------------------------------------------------------------------------------------------------

def grid(nx, ny, v0=0):
    """(nx-1)(ny-1)*2 faces over an nx x ny vertex grid starting at vertex v0: one cluster."""
    i, j = np.meshgrid(np.arange(nx - 1), np.arange(ny - 1), indexing="ij")
    a = (i * ny + j).ravel() + v0
    b, c, d = a + ny, a + 1, a + ny + 1
    return np.concatenate([np.stack([a, b, c], 1), np.stack([c, b, d], 1)]).astype(np.int64)


def bipyramid(n, v0=0):
    """A closed double cone of 2n faces over n rim vertices (v0 .. v0+n-1) and two apexes."""
    r = np.arange(n) + v0
    s = (np.arange(n) + 1) % n + v0
    top, bot = v0 + n, v0 + n + 1
    return np.concatenate([np.stack([r, s, np.full(n, top)], 1), np.stack([s, r, np.full(n, bot)], 1)]).astype(np.int64)


def fan(n, v0=0):
    """An open fan of n faces around vertex v0: one cluster of n faces."""
    r = np.arange(n) + v0 + 1
    return np.stack([np.full(n, v0), r, r + 1], 1).astype(np.int64)


def strip(n, v0=0):
    """A strip of n faces, each sharing an edge with the next: the longest chain (diameter n)."""
    i = np.arange(n) + v0
    return np.stack([i, i + 1, i + 2], 1).astype(np.int64)
