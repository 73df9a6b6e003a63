"""Drives libsurfel_b200.so stage by stage through the C ABI and exposes every intermediate as
numpy, so the parity tests can compare each one with the oracle (tests only)."""
import ctypes

import numpy as np
import torch

from diff_surfel_rasterization import _cabi


def _t(x, dtype=torch.float32):
    return None if x is None else torch.as_tensor(np.ascontiguousarray(x)).to(dtype).cuda().contiguous()


def _p(t):
    return None if t is None else t.data_ptr()


class CudaPipeline:
    def __init__(self, scene, cam, bg, sh_degree=3, scale_modifier=1.0, tile_rows=(0, 0), fused_count=True, lib=None):
        """lib: a library handle from _cabi.load_handle() (a test variant of the kernels); default the main library."""
        self.fused_count = fused_count
        self.lib = _cabi.load() if lib is None else lib
        self.W, self.H = cam["W"], cam["H"]
        self.gx, self.gy = (self.W + 15) // 16, (self.H + 15) // 16
        g = lambda k: scene.get(k)
        self.means3D = _t(g("means3D")); self.scales = _t(g("scales")); self.rotations = _t(g("rotations"))
        self.opacities = _t(g("opacities")); self.shs = _t(g("shs"))
        self.transMat_precomp = _t(g("transMat_precomp")); self.colors_precomp = _t(g("colors_precomp"))
        self.bg = _t(bg); self.vm = _t(cam["viewmatrix"]); self.pm = _t(cam["projmatrix"]); self.campos = _t(cam["campos"])
        self.P = self.means3D.shape[0]
        self.M = 0 if self.shs is None else self.shs.shape[1]
        self.cs = _cabi.SurfelSettings(self.H, self.W, float(cam["tanfovx"]), float(cam["tanfovy"]),
                                       float(scale_modifier), int(sh_degree), 0, 0, int(tile_rows[0]), int(tile_rows[1]),
                                       self.bg.data_ptr(), self.vm.data_ptr(), self.pm.data_ptr(), self.campos.data_ptr())
        self.stream = torch.cuda.current_stream().cuda_stream

    def _check(self, status):
        _cabi.check(status, self.lib)

    # ---- stage 1 ----
    def preprocess(self):
        lib, P = self.lib, self.P
        # workspaces are handed over UNINITIALISED by the product (torch.empty): poison them here so that a
        # kernel reading a byte it did not write first cannot pass
        self.radii = torch.full((P,), -1, dtype=torch.int32, device="cuda")
        self.geom = torch.full((lib.surfel_geom_bytes(P),), 0xFF, dtype=torch.uint8, device="cuda")
        self.img = torch.full((lib.surfel_image_bytes(self.W, self.H),), 0xFF, dtype=torch.uint8, device="cuda")
        host_R = torch.zeros(1, dtype=torch.int32).pin_memory()
        self._check(lib.surfel_forward_preprocess(
            ctypes.byref(self.cs), P, self.M, _p(self.means3D), _p(self.opacities), _p(self.scales),
            _p(self.rotations), _p(self.transMat_precomp), _p(self.shs), _p(self.colors_precomp),
            self.radii.data_ptr(), self.geom.data_ptr(), self.img.data_ptr() if self.fused_count else None,
            host_R.data_ptr(), self.stream))
        torch.cuda.synchronize()
        self.R = int(host_R.item()) & 0xFFFFFFFF
        offs = (ctypes.c_size_t * 6)()
        lib.surfel_geom_offsets(P, offs)
        g = self.geom.cpu().numpy()
        rec = g[offs[0]:offs[0] + P * 128].view(np.float32).reshape(P, 32)     # render record (common.cuh)
        tmr = g[offs[5]:offs[5] + P * 48].view(np.float32).reshape(P, 12)      # transform record
        out = dict(
            radii=self.radii.cpu().numpy(),
            tiles_touched=g[offs[1]:offs[1] + 4 * P].view(np.uint32).copy(),
            offsets=g[offs[2]:offs[2] + 4 * P].view(np.uint32).copy(),
            clamped_bits=g[offs[3]:offs[3] + P].copy(),
            transMat=tmr[:, 0:9].copy(), xy=tmr[:, 9:11].copy(), depths=tmr[:, 11].copy(),
            opacity=rec[:, 11].copy(), normal=rec[:, 12:15].copy(), rgb=rec[:, 16:19].copy(),
            adjugate=rec[:, [0, 1, 2, 4, 5, 6, 8, 9, 10]].copy(), det=rec[:, 19].copy(),
            bbox=rec[:, 24:28].copy(), diag=rec[:, 28:32].copy(), R=self.R)
        out["clamped"] = np.stack([(out["clamped_bits"] >> c) & 1 for c in range(3)], 1).astype(np.uint8)
        return out

    # ---- stage 2 ----
    def _bin_views(self):
        offs = (ctypes.c_size_t * 5)()
        self.lib.surfel_binning_offsets(self.R, self.W, self.H, offs)
        return list(offs)

    def duplicate(self):
        lib = self.lib
        self.binning = torch.full((lib.surfel_binning_bytes(self.R, self.W, self.H),), 0xFF, dtype=torch.uint8, device="cuda")
        self._check(lib.surfel_bin_duplicate(ctypes.byref(self.cs), self.P, self.R, self.geom.data_ptr(),
                                             self.radii.data_ptr(), self.binning.data_ptr(), self.stream))
        torch.cuda.synchronize()
        o = self._bin_views()
        b = self.binning.cpu().numpy()
        R = self.R
        return dict(keys_unsorted=b[o[0]:o[0] + 8 * R].view(np.uint64).copy(),
                    vals_unsorted=b[o[1]:o[1] + 4 * R].view(np.uint32).copy())

    def bucket(self):
        """Production binning path (tile buckets + per-tile sort); same outputs as duplicate()+sort()."""
        lib = self.lib
        self.binning = torch.full((lib.surfel_binning_bytes(self.R, self.W, self.H),), 0xFF, dtype=torch.uint8, device="cuda")
        self._check(lib.surfel_bin_bucket(ctypes.byref(self.cs), self.P, self.R, self.geom.data_ptr(),
                                          self.radii.data_ptr(), self.binning.data_ptr(),
                                          self.img.data_ptr() if self.fused_count else None, 1, self.stream))
        torch.cuda.synchronize()
        o = self._bin_views()
        b = self.binning.cpu().numpy()
        R, tiles = self.R, self.gx * self.gy
        return dict(keys_sorted=b[o[2]:o[2] + 8 * R].view(np.uint64).copy(),
                    vals_sorted=b[o[3]:o[3] + 4 * R].view(np.uint32).copy(),
                    ranges=b[o[4]:o[4] + 8 * tiles].view(np.uint32).reshape(tiles, 2).copy())

    def sort(self):
        self._check(self.lib.surfel_bin_sort(ctypes.byref(self.cs), self.R, self.binning.data_ptr(), self.stream))
        torch.cuda.synchronize()
        o = self._bin_views()
        b = self.binning.cpu().numpy()
        R, tiles = self.R, self.gx * self.gy
        return dict(keys_sorted=b[o[2]:o[2] + 8 * R].view(np.uint64).copy(),
                    vals_sorted=b[o[3]:o[3] + 4 * R].view(np.uint32).copy(),
                    ranges=b[o[4]:o[4] + 8 * tiles].view(np.uint32).reshape(tiles, 2).copy())

    def render(self):
        lib, W, H = self.lib, self.W, self.H
        band = self.cs.tile_row_begin != 0 or self.cs.tile_row_end != 0      # a band leaves the other rows untouched
        fill = 0.0 if band else float("nan")
        self.color = torch.full((3, H, W), fill, device="cuda"); self.others = torch.full((7, H, W), fill, device="cuda")
        self._check(lib.surfel_render_forward(ctypes.byref(self.cs), self.R, self.geom.data_ptr(),
                                              self.binning.data_ptr(), self.img.data_ptr(),
                                              self.color.data_ptr(), self.others.data_ptr(), self.stream))
        torch.cuda.synchronize()
        offs = (ctypes.c_size_t * 2)()
        lib.surfel_image_offsets(W, H, offs)
        i = self.img.cpu().numpy()
        n = W * H
        return dict(color=self.color.cpu().numpy(), others=self.others.cpu().numpy(),
                    accum=i[offs[0]:offs[0] + 12 * n].view(np.float32).reshape(3, H, W).copy(),
                    n_contrib=i[offs[1]:offs[1] + 8 * n].view(np.uint32).reshape(2, H, W).copy())

    def backward(self, dL_dcolor, dL_dothers, lowpass_quirk=True, defer_sh=False):
        """defer_sh: surfel_settings.sh_grad_deferred = 1 (dL_dsh left to surfel_sh_grad_expand, which is then
        run here on the kernel's clamp-masked colour gradients; dL_dshs is poisoned first, so a row the expansion
        misses cannot pass)."""
        lib, P, M = self.lib, self.P, self.M
        self.cs.sh_grad_deferred = int(bool(defer_sh))
        gc, go = _t(dL_dcolor), _t(dL_dothers)
        e = lambda *s: torch.full(s, float("nan"), device="cuda")
        scratch = e(max(P, 1), lib.surfel_grad_scratch_floats())
        out = dict(dL_dmeans2D=e(P, 3), dL_dcolors=e(P, 3), dL_dopacity=e(P, 1), dL_dmeans3D=e(P, 3),
                   dL_dtransMat=e(P, 9), dL_dshs=e(P, max(M, 1), 3), dL_dscales=e(P, 2), dL_drotations=e(P, 4))
        self._check(lib.surfel_backward(
            ctypes.byref(self.cs), P, M, self.R, _p(self.means3D), _p(self.scales), _p(self.rotations),
            _p(self.transMat_precomp), _p(self.shs), int(self.colors_precomp is not None),
            self.radii.data_ptr(), self.geom.data_ptr(), self.binning.data_ptr(), self.img.data_ptr(),
            gc.data_ptr(), go.data_ptr(), scratch.data_ptr(), out["dL_dmeans2D"].data_ptr(),
            out["dL_dcolors"].data_ptr(), out["dL_dopacity"].data_ptr(), out["dL_dmeans3D"].data_ptr(),
            out["dL_dtransMat"].data_ptr(), out["dL_dshs"].data_ptr() if M else None,
            out["dL_dscales"].data_ptr() if self.scales is not None else None,
            out["dL_drotations"].data_ptr() if self.rotations is not None else None,
            int(lowpass_quirk), self.stream))
        self.cs.sh_grad_deferred = 0
        if defer_sh and M:
            self._check(lib.surfel_sh_grad_expand(P, M, int(self.cs.sh_degree), self.means3D.data_ptr(), self.campos.data_ptr(),
                                                  out["dL_dcolors"].data_ptr(), out["dL_dshs"].data_ptr(), self.stream))
        torch.cuda.synchronize()
        res = {k: v.cpu().numpy() for k, v in out.items()}
        res["grad_rec"] = scratch.cpu().numpy()
        return res
