"""ctypes/numpy front-end of the CPU oracle (oracle/surfel_oracle.c).

TEST INFRASTRUCTURE ONLY — see the header of surfel_oracle.c.  Imported by tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs; never by the
product package.  PARITY UNPINNED for the rasterizer proper (no reference source, no reference
tests); the T-matrix / SH / camera conventions are pinned by tests/golden.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libsurfel_oracle.so")
_lib = None

BLOCK = 16


def build(force=False):
    """Compile libsurfel_oracle.so with gcc (building the checker is not using it)."""
    src = os.path.join(_HERE, "surfel_oracle.c")
    if (not force and os.path.exists(_LIB_PATH)
            and os.path.getmtime(_LIB_PATH) >= os.path.getmtime(src)):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-B", "libsurfel_oracle.so"],
                          stdout=subprocess.DEVNULL)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = ctypes.CDLL(_LIB_PATH)
        _lib.oracle_scan.restype = ctypes.c_uint32
        _lib.oracle_tile_bits.restype = ctypes.c_int
    return _lib


def set_threads(n=0):
    """OpenMP threads used by the oracle's parallel loops (0 = every core); returns the count in force."""
    return int(lib().oracle_set_threads(int(n)))


def _p(a):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ctypes.c_void_p)


def _f32(a):
    return None if a is None else np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def grid(W, H):
    return (W + BLOCK - 1) // BLOCK, (H + BLOCK - 1) // BLOCK


def tile_bits(n):
    return lib().oracle_tile_bits(ctypes.c_uint(n))


def preprocess_fwd(means3D, scales, rotations, opacities, shs, viewmatrix, projmatrix, campos,
                   W, H, sh_degree=3, scale_modifier=1.0, transMat_precomp=None,
                   colors_precomp=None, row0=0, row1=None):
    means3D = _f32(means3D)
    P = means3D.shape[0]
    gx, gy = grid(W, H)
    row1 = gy if row1 is None else row1
    scales, rotations, opacities = _f32(scales), _f32(rotations), _f32(opacities).reshape(-1)
    shs = _f32(shs)
    M = 0 if shs is None else shs.shape[1]
    out = dict(
        radii=np.zeros(P, np.int32), xy=np.zeros((P, 2), np.float32),
        depths=np.zeros(P, np.float32), transMat=np.zeros((P, 9), np.float32),
        normal_opacity=np.zeros((P, 4), np.float32), rgb=np.zeros((P, 3), np.float32),
        clamped=np.zeros((P, 3), np.uint8), tiles_touched=np.zeros(P, np.uint32))
    tp, cp = _f32(transMat_precomp), _f32(colors_precomp)
    vm, pm, cam = _f32(viewmatrix).reshape(-1), _f32(projmatrix).reshape(-1), _f32(campos)
    lib().oracle_preprocess_fwd(
        P, int(sh_degree), M, _p(means3D), _p(scales), ctypes.c_float(scale_modifier),
        _p(rotations), _p(opacities), _p(shs), _p(tp), _p(cp), _p(vm), _p(pm), _p(cam),
        W, H, row0, row1, _p(out["radii"]), _p(out["xy"]), _p(out["depths"]), _p(out["transMat"]),
        _p(out["normal_opacity"]), _p(out["rgb"]), _p(out["clamped"]), _p(out["tiles_touched"]))
    return out


def mark_visible(means3D, viewmatrix):
    means3D = _f32(means3D)
    out = np.zeros(means3D.shape[0], np.uint8)
    lib().oracle_mark_visible(means3D.shape[0], _p(means3D), _p(_f32(viewmatrix).reshape(-1)), _p(out))
    return out.astype(bool)


def bin_sort(pre, W, H, row0=0, row1=None):
    gx, gy = grid(W, H)
    row1 = gy if row1 is None else row1
    P = pre["radii"].shape[0]
    offsets = np.zeros(P, np.uint32)
    R = int(lib().oracle_scan(P, _p(pre["tiles_touched"]), _p(offsets)))
    out = dict(offsets=offsets, R=R,
               keys_unsorted=np.zeros(R, np.uint64), vals_unsorted=np.zeros(R, np.uint32),
               keys_sorted=np.zeros(R, np.uint64), vals_sorted=np.zeros(R, np.uint32),
               ranges=np.zeros((gx * gy, 2), np.uint32))
    lib().oracle_bin(P, W, H, row0, row1, _p(pre["xy"]), _p(pre["depths"]), _p(pre["radii"]),
                     _p(offsets), ctypes.c_uint32(R), _p(out["keys_unsorted"]), _p(out["vals_unsorted"]),
                     _p(out["keys_sorted"]), _p(out["vals_sorted"]), _p(out["ranges"]))
    return out


def render_fwd(pre, binned, bg, W, H, f64=False):
    """A.3.  f64=True evaluates the same algorithm in double on the same float32 inputs (the exact value
    of the published formula; the yardstick for float32 rounding noise, not a parity target)."""
    out = dict(color=np.zeros((3, H, W), np.float32), others=np.zeros((7, H, W), np.float32),
               accum=np.zeros((3, H, W), np.float32), n_contrib=np.zeros((2, H, W), np.uint32))
    fn = lib().oracle_render_fwd_f64 if f64 else lib().oracle_render_fwd
    fn(W, H, _p(binned["ranges"]), _p(binned["vals_sorted"]), _p(pre["xy"]),
                            _p(pre["transMat"]), _p(pre["normal_opacity"]), _p(pre["rgb"]),
                            _p(_f32(bg)), _p(out["color"]), _p(out["others"]), _p(out["accum"]),
                            _p(out["n_contrib"]))
    return out


ABS_LAYOUT = (("dL_dtransMat", 0, 9), ("dL_dmean2D", 9, 11), ("dL_dopacity", 11, 12), ("dL_dnormal", 12, 15),
              ("dL_dcolors", 15, 18))


def render_bwd(pre, binned, img, bg, dL_dcolor, dL_dothers, W, H, lowpass_quirk=True, f64=False):
    """A.4.  f64=True: the per-pair arithmetic in double (yardstick for float32 rounding noise, not a parity target).
    With f64=True the result also holds out["abs"][key]: per entry, the sum of the absolute per-pair contributions."""
    P = pre["radii"].shape[0]
    out = dict(dL_dtransMat=np.zeros((P, 9), np.float64), dL_dmean2D=np.zeros((P, 2), np.float64),
               dL_dopacity=np.zeros(P, np.float64), dL_dnormal=np.zeros((P, 3), np.float64),
               dL_dcolors=np.zeros((P, 3), np.float64))
    args = [W, H, _p(binned["ranges"]), _p(binned["vals_sorted"]), _p(pre["xy"]),
            _p(pre["transMat"]), _p(pre["normal_opacity"]), _p(pre["rgb"]),
            _p(_f32(bg)), _p(img["accum"]), _p(img["n_contrib"]),
            _p(_f32(dL_dcolor)), _p(_f32(dL_dothers)), int(bool(lowpass_quirk)),
            _p(out["dL_dtransMat"]), _p(out["dL_dmean2D"]), _p(out["dL_dopacity"]),
            _p(out["dL_dnormal"]), _p(out["dL_dcolors"])]
    if f64:
        absum = np.zeros((P, 18), np.float64)
        lib().oracle_render_bwd_f64(*args, _p(absum))
        out["abs"] = {k: absum[:, a:b].reshape(out[k].shape) for k, a, b in ABS_LAYOUT}
    else:
        lib().oracle_render_bwd(*args)
    return out


MARGIN_NAMES = ("alpha_min", "alpha_clamp", "rho_branch", "near", "t_min", "median", "pz", "power")


def decision_margins(pre, binned, W, H, slack=1e-3):
    """Per-pixel smallest relative distance of any evaluated (pixel, splat) pair to each discontinuity of A.3, in
    float64 (oracle_decision_margins).  Returns (dict name -> (H, W) array, per-splat smallest margin (P,))."""
    P = pre["radii"].shape[0]
    m = np.zeros((len(MARGIN_NAMES), H, W), np.float64)
    per_splat = np.zeros(P, np.float64)
    lib().oracle_decision_margins(W, H, P, _p(binned["ranges"]), _p(binned["vals_sorted"]), _p(pre["xy"]),
                                  _p(pre["transMat"]), _p(pre["normal_opacity"]), ctypes.c_double(slack),
                                  _p(m), _p(per_splat))
    return dict(zip(MARGIN_NAMES, m)), per_splat


def preprocess_bwd(means3D, scales, rotations, shs, pre, rb, viewmatrix, projmatrix, campos, W, H,
                   sh_degree=3, scale_modifier=1.0, transMat_precomp=None, colors_precomp=None):
    means3D = _f32(means3D)
    P = means3D.shape[0]
    shs = _f32(shs)
    M = 0 if shs is None else shs.shape[1]
    gT = np.ascontiguousarray(rb["dL_dtransMat"].astype(np.float32))
    gm2 = np.zeros((P, 3), np.float32)
    gm2[:, :2] = rb["dL_dmean2D"].astype(np.float32)
    out = dict(dL_dtransMat=gT, dL_dmeans2D=gm2,
               dL_dmeans3D=np.zeros((P, 3), np.float32), dL_dscales=np.zeros((P, 2), np.float32),
               dL_drotations=np.zeros((P, 4), np.float32),
               dL_dshs=np.zeros((P, max(M, 1), 3), np.float32),
               dL_dopacity=rb["dL_dopacity"].astype(np.float32).reshape(P, 1),
               dL_dcolors=rb["dL_dcolors"].astype(np.float32))
    gn = np.ascontiguousarray(rb["dL_dnormal"].astype(np.float32))
    gc = np.ascontiguousarray(rb["dL_dcolors"].astype(np.float32))
    tp = _f32(transMat_precomp)
    lib().oracle_preprocess_bwd(
        P, int(sh_degree), M, _p(means3D), _p(_f32(scales)), ctypes.c_float(scale_modifier),
        _p(_f32(rotations)), _p(shs), _p(pre["clamped"]), _p(tp), int(colors_precomp is not None),
        _p(pre["radii"]), _p(pre["transMat"]), _p(_f32(viewmatrix).reshape(-1)),
        _p(_f32(projmatrix).reshape(-1)), _p(_f32(campos)), W, H, _p(gT), _p(gn), _p(gc), _p(gm2),
        _p(out["dL_dmeans3D"]), _p(out["dL_dscales"]), _p(out["dL_drotations"]), _p(out["dL_dshs"]))
    return out


def forward(scene, cam, bg, sh_degree=3, scale_modifier=1.0, row0=0, row1=None):
    """Full A.1-A.3 forward on a scene dict (see tests/scenes.py). Returns (pre, binned, img)."""
    W, H = cam["W"], cam["H"]
    pre = preprocess_fwd(scene["means3D"], scene.get("scales"), scene.get("rotations"),
                         scene["opacities"], scene.get("shs"), cam["viewmatrix"], cam["projmatrix"],
                         cam["campos"], W, H, sh_degree, scale_modifier,
                         scene.get("transMat_precomp"), scene.get("colors_precomp"), row0, row1)
    binned = bin_sort(pre, W, H, row0, row1)
    img = render_fwd(pre, binned, bg, W, H)
    return pre, binned, img


def backward(scene, cam, bg, pre, binned, img, dL_dcolor, dL_dothers, sh_degree=3,
             scale_modifier=1.0, lowpass_quirk=True, f64=False):
    W, H = cam["W"], cam["H"]
    rb = render_bwd(pre, binned, img, bg, dL_dcolor, dL_dothers, W, H, lowpass_quirk, f64)
    return preprocess_bwd(scene["means3D"], scene.get("scales"), scene.get("rotations"),
                          scene.get("shs"), pre, rb, cam["viewmatrix"], cam["projmatrix"],
                          cam["campos"], W, H, sh_degree, scale_modifier,
                          scene.get("transMat_precomp"), scene.get("colors_precomp"))
