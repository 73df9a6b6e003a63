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
No CPU path.
"""
import torch

from . import _cabi


def _side_ok(n):
    return 1 <= n <= (1 << 24)


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
