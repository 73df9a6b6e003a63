"""Cluster filtering of an extracted mesh on the device: `post_process_mesh` returns what the reference's
`post_process_mesh` (utils/mesh_utils.py:22-43, the last step of every mesh `render.py` exports) leaves in the Open3D
mesh it returns, computed from the CUDA tensors `UnboundedTSDF.extract_mesh` returns (csrc/meshpost.cu):

    verts, faces = field.extract_mesh(N, R)
    rgbs = field.colors(verts)
    verts, faces, rgbs = post_process_mesh(verts, faces, rgbs, cluster_to_keep=args.num_cluster)   # render.py:106

Rules and quirks (Python indexing of the k-th largest count, the floor of 50 faces, degenerate faces dropped after
unreferenced vertices): DESIGN.md §7k.  No CPU path.
"""
import torch

from . import _cabi

MAX_VERTS = 1 << 31          # vertex indices travel in 32 bits
MAX_RECORDS = 1 << 30        # 3 F edge records: the radix sort's limit


def threshold_index(cluster_to_keep, n_clusters):
    """The position np.sort(counts)[-cluster_to_keep] reads in an array of n_clusters counts, with Python's rules:
    k = 0 reads the smallest, a negative k counts from the bottom, and IndexError when it falls outside."""
    i = -int(cluster_to_keep)
    j = i + n_clusters if i < 0 else i
    if not 0 <= j < n_clusters:
        raise IndexError(f"index {i} is out of bounds for axis 0 with size {n_clusters}")
    return j


def _check(verts, faces, colors, cluster_to_keep):
    import numpy as np
    who = "post_process_mesh"
    if isinstance(cluster_to_keep, bool) or not isinstance(cluster_to_keep, (int, np.integer)):
        raise RuntimeError(f"{who}: cluster_to_keep must be an integer, got {cluster_to_keep!r}")
    for name, t in (("verts", verts), ("faces", faces), ("colors", colors)):
        if t is None and name == "colors":
            continue
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise RuntimeError(f"{who}: {name} must be a CUDA tensor (there is no CPU path)")
    if verts.dtype != torch.float32 or verts.dim() != 2 or verts.shape[1] != 3:
        raise RuntimeError(f"{who}: verts must be (M,3) float32, got {tuple(verts.shape)} {verts.dtype}")
    if faces.dtype not in (torch.int64, torch.int32) or faces.dim() != 2 or faces.shape[1] != 3:
        raise RuntimeError(f"{who}: faces must be (F,3) int64 or int32, got {tuple(faces.shape)} {faces.dtype}")
    if faces.device != verts.device:
        raise RuntimeError(f"{who}: faces are on {faces.device}, verts on {verts.device}")
    if colors is not None:
        if colors.dim() != 2 or colors.shape[0] != verts.shape[0]:
            raise RuntimeError(f"{who}: colors must be (M,C) with M = {verts.shape[0]}, got {tuple(colors.shape)}")
        if colors.device != verts.device:
            raise RuntimeError(f"{who}: colors are on {colors.device}, verts on {verts.device}")
    M, F = verts.shape[0], faces.shape[0]
    if M >= MAX_VERTS:
        raise RuntimeError(f"{who}: {M} vertices; fewer than 2^31 are supported")
    if 3 * F >= MAX_RECORDS:
        raise RuntimeError(f"{who}: {F} faces give {3 * F} edge records; the radix sort takes fewer than 2^30")
    return M, F


@torch.no_grad()
def post_process_mesh(verts, faces, colors=None, cluster_to_keep=1000):
    """Removes the faces of every edge-connected cluster smaller than max(the cluster_to_keep-th largest cluster, 50)
    faces, then the vertices no kept face references, then the degenerate faces.  verts (M,3) float32 and faces (F,3)
    int64 or int32 on one CUDA device, colors None or (M,C) there.  Returns (verts (M',3) float32, faces (F',3) int64,
    colors (M',C) or None), gathered bit for bit, in input order, on the current stream; the inputs are not changed.
    IndexError where the reference's np.sort(...)[-cluster_to_keep] raises one (also on a mesh without faces)."""
    M, F = _check(verts, faces, colors, cluster_to_keep)
    if F == 0:
        threshold_index(cluster_to_keep, 0)          # raises, as the reference does on an empty mesh
    dev = verts.device
    lib = _cabi.load()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        faces = faces.to(torch.int64).contiguous()
        ws_bytes = lib.surfel_meshpost_workspace_bytes(M, F)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        face_cluster = torch.empty(F, dtype=torch.int32, device=dev)
        cluster_count = torch.empty(F, dtype=torch.int32, device=dev)
        info = torch.empty(2, dtype=torch.int64, device=dev)
        _cabi.check(lib.surfel_meshpost_clusters(M, F, faces.data_ptr(), ws.data_ptr(), ws_bytes,
                                                 face_cluster.data_ptr(), cluster_count.data_ptr(), info.data_ptr(),
                                                 stream))
        n_clusters, bad = info.tolist()              # first read: C and the index check
        if bad:
            raise RuntimeError(f"post_process_mesh: a face index lies outside [0, {M})")
        index = threshold_index(cluster_to_keep, n_clusters)
        out_faces = torch.empty((F, 3), dtype=torch.int64, device=dev)
        vert_map = torch.empty(max(M, 1), dtype=torch.int64, device=dev)
        _cabi.check(lib.surfel_meshpost_compact(M, F, faces.data_ptr(), face_cluster.data_ptr(),
                                                cluster_count.data_ptr(), n_clusters, index, ws.data_ptr(), ws_bytes,
                                                out_faces.data_ptr(), vert_map.data_ptr(), info.data_ptr(), stream))
        del ws, face_cluster, cluster_count
        m, f = info.tolist()                         # second read: M' and F'
        vert_map = vert_map[:m]
        out_faces = out_faces[:f] if f == F else out_faces[:f].clone()
        return (verts.index_select(0, vert_map), out_faces,
                None if colors is None else colors.index_select(0, vert_map))
