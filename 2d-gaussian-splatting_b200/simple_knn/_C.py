"""simple_knn._C.distCUDA2: the scale initialisation of GaussianModel.create_from_pcd
(/root/reference/scene/gaussian_model.py:134-135).

distCUDA2(points) -> (P,) float32 on points' device: entry i is the mean of the squared distances from point i
to its three nearest other points, computed exactly and bit-reproducibly by `surfel_knn_mean_sq_dist`
(csrc/knn.cu; rules in DESIGN.md §7g).  Fewer than three finite other points: the mean over those that exist
(0 if none).  A row with a NaN or inf coordinate is nobody's neighbour and gets NaN.

Launches on the current stream of the input's device and does not synchronise.  There is no CPU path.
"""
import torch


def distCUDA2(points):
    if not isinstance(points, torch.Tensor):
        raise RuntimeError(f"distCUDA2: expected a torch.Tensor, got {type(points).__name__}")
    if not points.is_cuda:
        raise RuntimeError("distCUDA2: points must be a CUDA tensor (there is no CPU path)")
    if points.dtype != torch.float32:
        raise RuntimeError(f"distCUDA2: points must be float32, got {points.dtype}")
    if points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError(f"distCUDA2: points must have shape (P, 3), got {tuple(points.shape)}")
    from diff_surfel_rasterization import _cabi
    lib = _cabi.load()
    dev = points.device
    P = points.shape[0]
    with torch.cuda.device(dev):
        out = torch.empty(P, dtype=torch.float32, device=dev)
        if P == 0:
            return out
        xyz = points.contiguous()
        nbytes = lib.surfel_knn_workspace_bytes(P)
        if nbytes == 0:
            raise RuntimeError(f"distCUDA2: {P} points exceed the supported count (2^30 - 1)")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _cabi.check(lib.surfel_knn_mean_sq_dist(P, xyz.data_ptr(), out.data_ptr(), ws.data_ptr(), nbytes,
                                                torch.cuda.current_stream(dev).cuda_stream))
    return out
