"""Fused TSDF evaluation for unbounded mesh extraction: `UnboundedTSDF` returns what the reference's
`compute_unbounded_tsdf` (utils/mesh_utils.py:197-248, used by `GaussianExtractor.extract_mesh_unbounded`,
`render.py --unbounded`) returns, with one CUDA launch per call (csrc/tsdf.cu) instead of a loop over the frames:

    field = UnboundedTSDF(self.depthmaps, self.rgbmaps, self.viewpoint_stack, self.center, self.radius, voxel_size)
    sdf_function = field                                                                # mesh_utils.py:258
    ...
    rgbs = field.colors(torch.tensor(np.asarray(mesh.vertices)).float().cuda())         # mesh_utils.py:277

The depth maps are uploaded once, at construction, and stay on the device for every call; the RGB maps are uploaded
on the first `colors()` call, so the field pass does not hold them.  Maps are (1,H,W) depth and (3,H,W) RGB tensors,
on the CPU or a CUDA device, and frames may differ in size; the cameras need `.full_proj_transform` (4,4).  The
device is `center`'s when it is a CUDA tensor, else the current CUDA device.  Rules and quirks: DESIGN.md §7i.
`extract_mesh(resolution, R)` replaces marching_cubes_with_contraction (mesh_utils.py:259-271) with marching cubes on
the device (csrc/mcubes.cu, DESIGN.md §7j).  No CPU path.
"""
import torch

from . import _cabi


CROP = 512          # the reference's cropN


def _side_ok(n):
    return 1 <= n <= (1 << 24)


def mesh_key_bits(side, n):
    """Bits of the largest vertex key of a grid of n^3 crops of side^3 points (csrc/mcubes.cu)."""
    G = (side - 1) * n + 1
    return (4 * G ** 3 - 1).bit_length()


def _mesh_crops(lib, stream, n, side, xs, center, radius, field):
    """Marching cubes over n^3 crops of side^3 points on `stream` (csrc/mcubes.cu).  Crop (i, j, k) spans
    [xs[i], xs[i+1]] x [xs[j], xs[j+1]] x [xs[k], xs[k+1]]; field(lib, bounds, out, stream) writes its side^3
    values to `out`.  center: 3 ctypes floats.  Returns (M,3) float32 vertices and (F,3) int64 faces."""
    dev = torch.device("cuda", torch.cuda.current_device())
    ws_bytes = lib.surfel_mcubes_crop_workspace_bytes(side)
    if ws_bytes == 0:
        raise RuntimeError(f"marching cubes: crop side {side} out of range")
    vol = torch.empty(side ** 3, dtype=torch.float32, device=dev)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    totals = torch.empty(2, dtype=torch.int64, device=dev)
    keys, pos, tris = [], [], []
    n_rec = 0
    for i in range(n):
        for j in range(n):
            for k in range(n):
                bounds = (_cabi.ctypes.c_double * 6)(xs[i], xs[i + 1], xs[j], xs[j + 1], xs[k], xs[k + 1])
                crop = (_cabi.c_int * 3)(i, j, k)
                field(lib, bounds, vol, stream)
                _cabi.check(lib.surfel_mcubes_crop_count(side, vol.data_ptr(), crop, n, ws.data_ptr(), ws_bytes,
                                                         totals.data_ptr(), stream.cuda_stream))
                nr, nt = totals.tolist()           # the crop's only device-to-host read
                n_rec += nr
                if n_rec >= 1 << 30:
                    raise RuntimeError(f"marching cubes: more than 2^30 vertex records ({n_rec} after crop "
                                       f"{(i, j, k)}), the limit of the radix sort")
                if nr == 0 and nt == 0:
                    continue
                kc = torch.empty(nr, dtype=torch.int64, device=dev)
                pc = torch.empty((nr, 3), dtype=torch.float32, device=dev)
                tc = torch.empty((nt, 3), dtype=torch.int64, device=dev)
                _cabi.check(lib.surfel_mcubes_crop_emit(side, vol.data_ptr(), bounds, crop, n, ws.data_ptr(),
                                                        ws_bytes, nr, nt, kc.data_ptr(), pc.data_ptr(),
                                                        tc.data_ptr(), stream.cuda_stream))
                keys.append(kc), pos.append(pc), tris.append(tc)
    del vol, ws
    cat = lambda ts, shape, dt: torch.cat(ts) if ts else torch.empty(shape, dtype=dt, device=dev)
    keys, pos, tris = cat(keys, (0,), torch.int64), cat(pos, (0, 3), torch.float32), cat(tris, (0, 3), torch.int64)
    n_tri = tris.shape[0]
    m_bytes = lib.surfel_mcubes_merge_workspace_bytes(n_rec)
    ws = torch.empty(max(m_bytes, 1), dtype=torch.uint8, device=dev)
    verts = torch.empty((n_rec, 3), dtype=torch.float32, device=dev)
    faces = torch.empty((n_tri, 3), dtype=torch.int64, device=dev)
    _cabi.check(lib.surfel_mcubes_merge(n_rec, keys.data_ptr(), pos.data_ptr(), n_tri, tris.data_ptr(),
                                        mesh_key_bits(side, n), center, radius, ws.data_ptr(), m_bytes,
                                        verts.data_ptr(), faces.data_ptr(), totals.data_ptr(), stream.cuda_stream))
    m = int(totals[0].item())
    return verts[:m], faces


class UnboundedTSDF:
    def __init__(self, depthmaps, rgbmaps, cameras, center, radius, voxel_size):
        depthmaps, cameras = list(depthmaps), list(cameras)
        rgbmaps = None if rgbmaps is None else list(rgbmaps)
        if len(depthmaps) != len(cameras):
            raise RuntimeError(f"UnboundedTSDF: {len(depthmaps)} depth maps for {len(cameras)} cameras")
        if rgbmaps is not None and len(rgbmaps) != len(cameras):
            raise RuntimeError(f"UnboundedTSDF: {len(rgbmaps)} RGB maps for {len(cameras)} cameras")
        c = torch.as_tensor(center).detach().to("cpu", torch.float32).reshape(-1)
        if c.numel() != 3:
            raise RuntimeError(f"UnboundedTSDF: center must hold 3 values, got {c.numel()}")
        self.center = (_cabi.c_float * 3)(*c.tolist())
        self.radius = float(radius)
        self.trunc = 5 * float(voxel_size)        # the double the reference forms; the kernel rounds it to float32

        V = len(cameras)
        self.frames = (_cabi.TsdfFrame * max(V, 1))()
        offset = 0
        for f, (cam, d) in enumerate(zip(cameras, depthmaps)):
            m = getattr(cam, "full_proj_transform", None)
            if not isinstance(m, torch.Tensor) or tuple(m.shape) != (4, 4):
                raise RuntimeError(f"UnboundedTSDF: camera {f} has no (4,4) full_proj_transform")
            if not isinstance(d, torch.Tensor) or d.dim() != 3 or d.shape[0] != 1:
                raise RuntimeError(f"UnboundedTSDF: depth map {f} must be a (1,H,W) tensor")
            H, W = int(d.shape[1]), int(d.shape[2])
            if not (_side_ok(H) and _side_ok(W)):
                raise RuntimeError(f"UnboundedTSDF: depth map {f} is {H}x{W}; each side must be in [1, 2^24]")
            if rgbmaps is not None:
                rm = rgbmaps[f]
                if not isinstance(rm, torch.Tensor) or tuple(rm.shape) != (3, H, W):
                    shape = tuple(rm.shape) if isinstance(rm, torch.Tensor) else type(rm).__name__
                    raise RuntimeError(f"UnboundedTSDF: RGB map {f} is {shape}, its depth map (1,{H},{W})")
            fr = self.frames[f]
            fr.full_proj_transform[:] = m.detach().to("cpu", torch.float32).reshape(-1).tolist()
            fr.height, fr.width, fr.offset = H, W, offset
            offset += H * W
        self.n_frames, self.map_pixels = V, offset
        if isinstance(center, torch.Tensor) and center.is_cuda:
            self.device = center.device
        else:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._rgbmaps = rgbmaps
        self._rgb = None
        with torch.cuda.device(self.device):
            self.depth, self._depth_ready = self._upload(depthmaps, 1)

    def _upload(self, maps, channels):
        """The maps concatenated in frame order into one float32 buffer on the device, copied map by map on the
        current stream, and an event recorded after them, which the stream of every call that reads them waits for."""
        buf = torch.empty(max(channels * self.map_pixels, 1), dtype=torch.float32, device=self.device)
        o = 0
        for m in maps:
            n = m.numel()
            buf[o:o + n].view(m.shape).copy_(m.detach())
            o += n
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(self.device))
        return buf, ready

    def _points(self, points, who):
        if not isinstance(points, torch.Tensor) or not points.is_cuda:
            raise RuntimeError(f"UnboundedTSDF.{who}: points must be a CUDA tensor (there is no CPU path)")
        if points.dtype != torch.float32:
            raise RuntimeError(f"UnboundedTSDF.{who}: points must be float32, got {points.dtype}")
        if points.dim() != 2 or points.shape[1] != 3:
            raise RuntimeError(f"UnboundedTSDF.{who}: points must be (N,3), got {tuple(points.shape)}")
        if points.device != self.device:
            raise RuntimeError(f"UnboundedTSDF.{who}: points are on {points.device}, the maps on {self.device}")
        return points.contiguous()

    def _eval(self, points, rgb, out):
        lib = _cabi.load()
        stream = torch.cuda.current_stream(self.device)
        stream.wait_event(self._depth_ready)
        if rgb is not None:
            stream.wait_event(self._rgb_ready)
        _cabi.check(lib.surfel_tsdf_eval(
            points.shape[0], points.data_ptr(), self.n_frames, self.frames, self.map_pixels, self.depth.data_ptr(),
            rgb.data_ptr() if rgb is not None else None, self.center, self.radius, self.trunc, out.data_ptr(),
            stream.cuda_stream))
        return out

    @torch.no_grad()
    def __call__(self, points):
        """(N,3) float32 points in contracted space -> (N,) float32 TSDF (mesh_utils.py:258)."""
        points = self._points(points, "__call__")
        with torch.cuda.device(self.device):
            out = torch.empty(points.shape[0], dtype=torch.float32, device=self.device)
            return self._eval(points, None, out)

    @torch.no_grad()
    def extract_mesh(self, resolution, R):
        """The isosurface of this field over [-R, R]^3 in contracted space at `resolution`^3 samples, as the
        reference's marching_cubes_with_contraction returns it (mesh_utils.py:259-271): (M,3) float32 world vertices
        (uncontracted, clipped to [-32, 32]) and (F,3) int64 faces, both on the field's device.  Crops of 512^3 are
        evaluated in grid mode and meshed on the device, one after another; rules: DESIGN.md §7j."""
        import math

        import numpy as np
        if isinstance(resolution, bool) or not isinstance(resolution, (int, np.integer)) \
                or resolution <= 0 or resolution % CROP:
            raise RuntimeError(f"UnboundedTSDF.extract_mesh: resolution {resolution!r} is not a positive multiple "
                               f"of {CROP}")
        R = float(R)
        if not (math.isfinite(R) and R > 0):
            raise RuntimeError(f"UnboundedTSDF.extract_mesh: R must be finite and > 0, got {R}")
        n = int(resolution) // CROP
        xs = np.linspace(-R, R, n + 1)
        lib = _cabi.load()
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device)
            stream.wait_event(self._depth_ready)
            return _mesh_crops(lib, stream, n, CROP, xs, self.center, self.radius, self._grid_field)

    def _grid_field(self, lib, bounds, out, stream):
        _cabi.check(lib.surfel_tsdf_eval_grid(CROP, bounds, self.n_frames, self.frames, self.map_pixels,
                                              self.depth.data_ptr(), self.center, self.radius, self.trunc,
                                              out.data_ptr(), stream.cuda_stream))

    @torch.no_grad()
    def colors(self, points):
        """(N,3) float32 world points -> (N,3) float32 running mean of the sampled RGB (mesh_utils.py:277)."""
        if self._rgbmaps is None:
            raise RuntimeError("UnboundedTSDF.colors: the field was built without RGB maps")
        points = self._points(points, "colors")
        with torch.cuda.device(self.device):
            if self._rgb is None:
                self._rgb, self._rgb_ready = self._upload(self._rgbmaps, 3)
            out = torch.empty((points.shape[0], 3), dtype=torch.float32, device=self.device)
            return self._eval(points, self._rgb, out)
