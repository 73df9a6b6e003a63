"""The capacity-launched forward and backward held to the exact-R pipeline.

`_RasterizeGaussians.forward` does not wait for the instance count R before it bins and renders: it launches with a
capacity remembered per (device, P, W, H, tile band) and only then reads R.  With slack (cap >= R) the frame it drew
is final and the backward runs with R = cap; with a clamped guess (cap < R) every range is clamped to cap, the frame
is wrong, and the wrapper re-launches into a fresh binning workspace with the tile counts preprocess left in the
image workspace.  This file holds each of those paths to the exact-R run:

  * stage level, slack: ranges, the point list inside them, keys, outputs, accum and n_contrib are BIT-equal to the
    exact-R run of the same preprocess, for cap in {R, R+1, R+255, 1.25 R + 4096, 2 R + 4096}, with the tile counts
    of preprocess and with the stand-alone count.  The binning workspace is zero-filled and splat 0 is made an opaque
    frame-covering splat, so a kernel that reads a slot at or beyond R draws it where it does not belong;
  * stage level, clamped: the call succeeds, writes nothing outside its binning workspace (4 KB guard bands on either
    side), leaves the geometry workspace and the per-tile counts byte-identical, clamps every range to cap, and a
    re-launch into the same image workspace and outputs is bit-equal to a fresh exact-R run.  The cut falls inside a
    tile of each sort class (warp <= 512, small <= 2048, large <= 16384, global);
  * backward at R = cap on the certified scenes of hitloop_scenes.py, held to the float64 evaluation with the
    no-budget bounds of test_hitloop_gpu.py, against the main library and every build.py variant;
  * through GaussianRasterizer and autograd: repeated calls, growth past the guess and back, an all-culled step,
    backward twice, band mode into caller-owned buffers and replicas, the radix-sort variant, and the bookkeeping
    of the capacity cache.  Each of these calls is bit-equal to the same call with the speculative launch off.
"""
import ctypes
import functools

import numpy as np
import pytest
import torch

import hitloop_scenes as HS
import surfel_scenes as S
from parity_bars import grad_check, record_stats
from test_hitloop_gpu import (FWD_TOL, GRAD_TOL, LEAF_KEYS, LEAF_TOL, LIBS, ROW_FLOOR, leaf_bound, leaf_jacobian_abs,
                              lib_handle, worst_ratio)
from test_hitloop_gpu import scene as hitloop_scene

pytestmark = pytest.mark.gpu

GUARD = 4096                      # guard band on either side of a binning workspace (a multiple of its 256 B alignment)
GUARD_PATTERN = np.arange(GUARD, dtype=np.int64) % 251      # not a multiple of a word: a shifted write shows
SENTINEL = -7.0                   # output entries the render must not write (rows outside a band)
CERTIFIED = ("count255", "count256", "count257", "count511", "count512", "count513", "count1100", "near_plane",
             "low_pass", "tile_band", "ragged49x33", "ragged41x1")
CROWDED = (700, 3000, 20000)      # entries per crowded tile: the small, large and global-memory sort classes
STAGE_SCENES = CERTIFIED + tuple(f"crowded{n}" for n in CROWDED)
SORT_CLASSES = (("warp", 1, 512), ("small", 513, 2048), ("large", 2049, 16384), ("global", 16385, 1 << 31))


def spec_cap(R):
    """The capacity the wrapper remembers after a call that saw R instances."""
    return int(R * 1.25) + 4096


# ---------------------------------------------------------------------------------------------- stage level
def crowded(per_tile):
    """test_bucket_sort_crowded_tiles' construction: thousands of small splats piled onto the four centre tiles of
    a 64x64 frame, a quarter of them at exactly equal depth."""
    W = H = 64
    cam = S.to_numpy(S.make_camera(W, H))
    rng = np.random.default_rng(per_tile)
    P = per_tile
    z = rng.uniform(3.0, 3.5, P).astype(np.float32)
    z[: P // 4] = np.float32(3.25)
    xy = rng.normal(0, 0.01, (P, 2)).astype(np.float32)
    scene = dict(means3D=np.concatenate([xy, z[:, None]], 1).astype(np.float32),
                 scales=np.full((P, 2), 0.004, np.float32),
                 rotations=np.tile(np.array([[1, 0, 0, 0]], np.float32), (P, 1)),
                 opacities=np.full((P, 1), 0.01, np.float32),
                 shs=rng.normal(0, 0.3, (P, 16, 3)).astype(np.float32))
    return scene, cam, np.zeros(3, np.float32), None


def stage_scene(O, name):
    """(scene, camera, background, tile band or None)."""
    if name.startswith("crowded"):
        return crowded(int(name[7:]))
    s = hitloop_scene(O, name)
    return s["scene"], s["cam"], HS.BG, s["rows"]


def poison_splat0(scene, cam):
    """Splat 0 becomes an opaque splat that covers the whole frame behind every other splat (std dev 400 px, opacity
    0.95).  Every slot of a zero-filled binning workspace names it: a kernel that reads a slot it should not blends
    it a second time, or where it does not belong, and the pixel changes."""
    s = {k: v.copy() for k, v in scene.items()}
    f = cam["W"] / (2.0 * cam["tanfovx"])
    z = 1.5 * float(s["means3D"][:, 2].max())
    s["means3D"][0] = (0.37 * z / f, 0.29 * z / f, z)
    s["scales"][0] = 400.0 * z / f
    s["rotations"][0] = (1.0, 0.0, 0.0, 0.0)
    s["opacities"][0] = 0.95
    return s


class Stage:
    """One preprocess (through tests/cuda_stages.py) and any number of capacity launches of binning + render on it,
    all through the C ABI, with guard-banded binning workspaces."""

    def __init__(self, scene, cam, bg, rows, lib=None):
        from cuda_stages import CudaPipeline
        self.pipe = p = CudaPipeline(scene, cam, bg, tile_rows=rows or (0, 0), lib=lib)
        p.preprocess()
        self.lib, self.W, self.H, self.R, self.P = p.lib, p.W, p.H, p.R, p.P
        self.tiles = p.gx * p.gy
        offs = (ctypes.c_size_t * 2)()
        self.lib.surfel_image_offsets(self.W, self.H, offs)
        self.nc_off = offs[1]
        # the image workspace is [accum | n_contrib | per-tile counts]; the counts start one aligned n_contrib after
        self.tc_off = offs[1] + -(-8 * self.W * self.H // 256) * 256
        assert self.lib.surfel_image_bytes(self.W, self.H) - self.tc_off == -(-4 * self.tiles // 256) * 256
        self.guard = torch.as_tensor(GUARD_PATTERN, dtype=torch.uint8).cuda()

    def tile_counts(self):
        return self.pipe.img[self.tc_off:]

    def outputs(self):
        H, W = self.H, self.W
        return torch.full((3, H, W), SENTINEL, device="cuda"), torch.full((7, H, W), SENTINEL, device="cuda")

    def workspace(self, cap):
        n = self.lib.surfel_binning_bytes(cap, self.W, self.H)
        buf = torch.zeros(n + 2 * GUARD, dtype=torch.uint8, device="cuda")
        buf[:GUARD] = self.guard
        buf[-GUARD:] = self.guard
        return buf, buf[GUARD:GUARD + n]

    def guards_intact(self, buf):
        return torch.equal(buf[:GUARD], self.guard) and torch.equal(buf[-GUARD:], self.guard)

    def views(self, ws, cap, n):
        """(ranges (tiles, 2) int64, first n slots of the point list, first n slots of the sorted keys) on the host."""
        offs = (ctypes.c_size_t * 5)()
        self.lib.surfel_binning_offsets(cap, self.W, self.H, offs)
        b = ws.cpu().numpy()
        return (b[offs[4]:offs[4] + 8 * self.tiles].view(np.uint32).reshape(-1, 2).astype(np.int64),
                b[offs[3]:offs[3] + 4 * cap].view(np.uint32)[:n].copy(),
                b[offs[2]:offs[2] + 8 * cap].view(np.uint64)[:n].copy())

    def launch(self, cap, ready, outs=None, reset_state=True):
        """surfel_forward_render with `cap` slots into a fresh zero-filled, guard-banded workspace.  The per-pixel
        state of the image workspace is poisoned first (reset_state) so that rows a band leaves alone compare equal."""
        p = self.pipe
        if reset_state:
            p.img[:self.tc_off] = 0xFF
        color, others = self.outputs() if outs is None else outs
        buf, ws = self.workspace(cap)
        p._check(self.lib.surfel_forward_render(ctypes.byref(p.cs), self.P, cap, p.radii.data_ptr(), p.geom.data_ptr(),
                                                ws.data_ptr(), p.img.data_ptr(), ready, color.data_ptr(),
                                                others.data_ptr(), p.stream))
        torch.cuda.synchronize()
        return dict(buf=buf, ws=ws, cap=cap, color=color, others=others, state=p.img[:self.tc_off].clone())

    def keys(self, cap, ready):
        """surfel_bin_bucket with write_keys = 1: (ranges, point list, keys) of the first R slots, and whether the
        slack slots of the point list and keys are still zero."""
        p = self.pipe
        buf, ws = self.workspace(cap)
        p._check(self.lib.surfel_bin_bucket(ctypes.byref(p.cs), self.P, cap, p.geom.data_ptr(), p.radii.data_ptr(),
                                            ws.data_ptr(), p.img.data_ptr() if ready else None, 1, p.stream))
        torch.cuda.synchronize()
        assert self.guards_intact(buf), f"cap {cap}: surfel_bin_bucket wrote outside its workspace"
        rg, pl, ks = self.views(ws, cap, cap)
        R = min(self.R, cap)
        return rg, pl[:R], ks[:R], bool((pl[R:] == 0).all() and (ks[R:] == 0).all())


def bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def same_frame(got, ref):
    """Names of the outputs, or of the per-pixel state the backward reads, that are not bit-equal."""
    return [k for k in ("color", "others", "state") if not torch.equal(bits(got[k]), bits(ref[k]))]


@pytest.mark.parametrize("name", STAGE_SCENES)
def test_slack_capacity_is_invisible(oracle, cuda_lib, name):
    sc, cam, bg, rows = stage_scene(oracle, name)
    st = Stage(poison_splat0(sc, cam), cam, bg, rows)
    R = st.R
    assert R > 0 and int(st.pipe.radii[0]) > 0, "the poisoned splat must be visible"
    ref = st.launch(R, 1)
    assert st.guards_intact(ref["buf"])
    ref_rg, ref_pl, _ = st.views(ref["ws"], R, R)
    assert ref_rg[:, 1].max() == R and (ref_rg[:, 1] - ref_rg[:, 0]).sum() == R
    k_rg, k_pl, k_ks, _ = st.keys(R, 1)
    np.testing.assert_array_equal(k_rg, ref_rg)
    np.testing.assert_array_equal(k_pl, ref_pl)
    failures = []
    for cap in sorted({R, R + 1, R + 255, spec_cap(R), 2 * R + 4096}):
        for ready in (1, 0):
            got = st.launch(cap, ready)
            rg, pl, _ = st.views(got["ws"], cap, cap)
            if not st.guards_intact(got["buf"]):
                failures.append(f"cap {cap} ready {ready}: write outside the binning workspace")
            if not np.array_equal(rg, ref_rg):
                failures.append(f"cap {cap} ready {ready}: ranges differ")
            if not np.array_equal(pl[:R], ref_pl):
                failures.append(f"cap {cap} ready {ready}: point list differs inside the ranges")
            if (pl[R:] != 0).any():
                failures.append(f"cap {cap} ready {ready}: a slack slot of the point list was written")
            bad = same_frame(got, ref)
            if bad:
                failures.append(f"cap {cap} ready {ready}: {bad} differ from the exact-R run")
            rg, pl, ks, slack_clean = st.keys(cap, ready)
            if not (np.array_equal(rg, k_rg) and np.array_equal(pl, k_pl) and np.array_equal(ks, k_ks) and slack_clean):
                failures.append(f"cap {cap} ready {ready}: surfel_bin_bucket(write_keys=1) differs from the exact-R run")
    assert not failures, f"{name} (R = {R}):\n" + "\n".join(failures)


def tile_cuts(ranges):
    """Capacities that cut the longest tile of each sort class present: one slot past its start, one before its
    end (the clamped part then stays in the tile's class)."""
    L = ranges[:, 1] - ranges[:, 0]
    cuts = {}
    for cls, lo, hi in SORT_CLASSES:
        sel = np.nonzero((L >= lo) & (L <= hi))[0]
        if sel.size:
            t = sel[np.argmax(L[sel])]
            cuts[cls] = {int(ranges[t, 0]) + 1, int(ranges[t, 1]) - 1}
    return cuts


@pytest.mark.parametrize("name", STAGE_SCENES)
def test_clamped_capacity_stays_in_bounds_and_relaunch_is_exact(oracle, cuda_lib, name):
    sc, cam, bg, rows = stage_scene(oracle, name)
    st = Stage(poison_splat0(sc, cam), cam, bg, rows)
    R = st.R
    ref = st.launch(R, 1)
    ref_rg, ref_pl, _ = st.views(ref["ws"], R, R)
    cuts = tile_cuts(ref_rg)
    if name.startswith("crowded"):
        expect = {700: "small", 3000: "large", 20000: "global"}[int(name[7:])]
        assert expect in cuts, f"no {expect}-class tile: {sorted(cuts)}"
    caps = {1, R // 3, R - 1}.union(*cuts.values())
    caps = sorted(c for c in caps if 0 < c < R)
    geom0, counts0 = st.pipe.geom.clone(), st.tile_counts().clone()
    failures = []
    for cap in caps:
        for cap2 in (R, spec_cap(R)):
            outs = st.outputs()
            got = st.launch(cap, 1, outs=outs)
            if not st.guards_intact(got["buf"]):
                failures.append(f"cap {cap}: write outside the binning workspace")
            if not torch.equal(st.pipe.geom, geom0):
                failures.append(f"cap {cap}: the geometry workspace changed")
            if not torch.equal(st.tile_counts(), counts0):
                failures.append(f"cap {cap}: the per-tile counts the re-launch reads changed")
            rg, pl, _ = st.views(got["ws"], cap, cap)
            clamped = np.minimum(ref_rg, cap)
            clamped[clamped[:, 0] == clamped[:, 1]] = 0
            if not np.array_equal(rg, clamped):
                failures.append(f"cap {cap}: ranges are not the exact ranges clamped to cap")
            whole = int(ref_rg[:, 1][ref_rg[:, 1] <= cap].max(initial=0))     # slots of the tiles below the cut
            if not np.array_equal(pl[:whole], ref_pl[:whole]):
                failures.append(f"cap {cap}: point list of the tiles below the cut differs")
            # same image workspace (with the counts preprocess left), same outputs, fresh binning workspace
            again = st.launch(cap2, 1, outs=outs, reset_state=False)
            bad = same_frame(again, ref)
            if bad or not st.guards_intact(again["buf"]):
                failures.append(f"cap {cap} -> re-launch at {cap2}: {bad} differ from a fresh exact-R run")
    assert len(caps) >= 3
    assert not failures, f"{name} (R = {R}, cuts {cuts}):\n" + "\n".join(failures)


def background_frame(st, got, bg, rows):
    """An empty frame: every range zero, colour = background, allmap = 0, final T = 1, no contributor."""
    H, W = st.H, st.W
    ys = slice(0, H) if rows is None else slice(rows[0] * 16, min(H, rows[1] * 16))
    rg, _, _ = st.views(got["ws"], got["cap"], 0)
    assert (rg == 0).all()
    assert st.guards_intact(got["buf"])
    bgt = torch.as_tensor(bg).cuda().view(3, 1, 1).expand(3, H, W)
    assert torch.equal(got["color"][:, ys], bgt[:, ys])
    assert bool((got["others"][:, ys] == 0).all())
    n = H * W
    state = got["state"]
    T = state[:4 * n].view(torch.float32).view(H, W)
    last = state[st.nc_off:st.nc_off + 4 * n].view(torch.int32).view(H, W)
    assert bool((T[ys] == 1.0).all()) and bool((last[ys] == 0).all())


def test_empty_capacity_and_empty_frames(oracle, cuda_lib):
    """cap = 0 with P > 0; everything culled (R = 0) with cap > 0; P = 0.  Each draws the background."""
    sc, cam, bg, rows = stage_scene(oracle, "count256")
    st = Stage(sc, cam, bg, rows)
    assert st.R > 0
    counts0 = st.tile_counts().clone()
    background_frame(st, st.launch(0, 1), bg, rows)
    assert torch.equal(st.tile_counts(), counts0)
    # everything behind the camera: preprocess culls every splat
    culled = {k: v.copy() for k, v in sc.items()}
    culled["means3D"][:, 2] = -1.0 - np.abs(culled["means3D"][:, 2])
    st = Stage(culled, cam, bg, rows)
    assert st.R == 0 and int(st.pipe.radii.abs().max()) == 0
    for cap in (0, 1, 4096):
        for ready in (1, 0):
            background_frame(st, st.launch(cap, ready), bg, rows)
    # P = 0: preprocess leaves no counts, so the wrapper launches with tile_counts_ready = 0
    empty = {k: v[:0].copy() for k, v in sc.items()}
    st = Stage(empty, cam, bg, rows)
    assert st.P == 0 and st.R == 0
    for cap in (0, 4096):
        background_frame(st, st.launch(cap, 0), bg, rows)


# ---------------------------------------------------------------------------------------------- backward at R = cap
@pytest.mark.parametrize("lib", LIBS)
@pytest.mark.parametrize("name", CERTIFIED)
def test_backward_with_slack_matches_exact_evaluation(oracle, cuda_lib, lib, name):
    """The binning workspace is laid out for 1.25 R + 4096 slots (zero-filled: a slack slot reads as splat 0) and
    the backward runs with R = cap.  Bounds and scenes as test_hitloop_gpu.py, with no budget."""
    from cuda_stages import CudaPipeline
    s = hitloop_scene(oracle, name)
    HS.assert_certified(s)
    sc, cam, pre, binned, img = s["scene"], s["cam"], s["pre"], s["binned"], s["img"]
    W, H, rows = cam["W"], cam["H"], s["rows"]
    pipe = CudaPipeline(sc, cam, HS.BG, tile_rows=rows or (0, 0), lib=lib_handle(cuda_lib, lib))
    pipe.preprocess()
    cap = spec_cap(pipe.R)
    bk = pipe.bucket(cap=cap, fill=0)
    np.testing.assert_array_equal(bk["ranges"], binned["ranges"])
    np.testing.assert_array_equal(bk["vals_sorted"], binned["vals_sorted"])
    gi = pipe.render(cap=cap)
    ys = slice(0, H) if rows is None else slice(rows[0] * 16, min(H, rows[1] * 16))
    np.testing.assert_array_equal(gi["n_contrib"][:, ys], img["n_contrib"][:, ys])
    failures = []
    for key, got, ref in (("color", gi["color"], img["color"]), ("others", gi["others"], img["others"]),
                          ("accum", gi["accum"], img["accum"])):
        g, r = got[:, ys].astype(np.float64), ref[:, ys].astype(np.float64)
        err = np.abs(g - r) / np.maximum(1.0, np.abs(r))
        st = record_stats(f"capacity fwd {key}", err, dict(tol=FWD_TOL, scene=name, lib=lib))
        if not (np.isfinite(g).all() and st["max"] <= FWD_TOL):
            failures.append(f"forward {key}: max rel error {st['max']:.3e} > {FWD_TOL}")
    jac = leaf_jacobian_abs(oracle, name, s)
    img_gpu = dict(accum=img["accum"].copy(), n_contrib=img["n_contrib"].copy())
    img_gpu["accum"][:, ys], img_gpu["n_contrib"][:, ys] = gi["accum"][:, ys], gi["n_contrib"][:, ys]
    for gi_, group in enumerate(HS.CHANNEL_GROUPS):
        gc, go = HS.cotangent(W, H, group, seed=gi_)
        if rows is not None:
            gc[:, :ys.start] = 0; go[:, :ys.start] = 0
        rb = oracle.render_bwd(pre, binned, img_gpu, HS.BG, gc, go, W, H, f64=True)
        ref = oracle.preprocess_bwd(sc["means3D"], sc["scales"], sc["rotations"], sc["shs"], pre, rb, cam["viewmatrix"],
                                    cam["projmatrix"], cam["campos"], W, H)
        got = pipe.backward(gc, go, cap=cap)
        rec = got["grad_rec"].astype(np.float64)
        for key, g in (("dL_dmean2D", rec[:, 13:15]), ("dL_dopacity", rec[:, 15]), ("dL_dnormal", rec[:, 16:19]),
                       ("dL_dcolors", rec[:, 19:22])):
            r, nz = worst_ratio(np.abs(g - rb[key]), rb["abs"][key])
            record_stats(f"capacity bwd {key} / abs-sum", np.array([r]), dict(tol=GRAD_TOL, scene=name, lib=lib, cot=group, nz=nz))
            if r > GRAD_TOL or nz or not np.isfinite(g).all():
                failures.append(f"{group}: render-level {key}: worst error / abs-sum {r:.3e} (nonzero where 0: {nz})")
        bound = leaf_bound(oracle, jac, rb["abs"])
        splat_scale = np.max([bound[k].reshape(bound[k].shape[0], -1).max(1) for k in LEAF_KEYS], 0)
        for key in LEAF_KEYS:
            g = got[key].astype(np.float64).reshape(ref[key].shape)
            rk, bk_ = ref[key], bound[key]
            if key == "dL_dmeans2D":
                g, rk, bk_ = g[:, :2], rk[:, :2], bk_[:, :2]
            bk_ = bk_ + ROW_FLOOR * splat_scale.reshape((-1,) + (1,) * (bk_.ndim - 1))
            r, nz = worst_ratio(np.abs(g - rk), bk_)
            record_stats(f"capacity leaf {key} / bound", np.array([r]), dict(tol=LEAF_TOL[key], scene=name, lib=lib, cot=group, nz=nz))
            if r > LEAF_TOL[key] or nz or not np.isfinite(g).all():
                failures.append(f"{group}: leaf {key}: worst error / bound {r:.3e} (nonzero where 0: {nz})")
    assert not failures, f"{name} [{lib}], cap {cap} for R {pipe.R}:\n" + "\n".join(failures)


# ---------------------------------------------------------------------------------------------- GaussianRasterizer
@pytest.fixture(autouse=True)
def fresh_capacity(monkeypatch):
    """Every test starts from an empty capacity table of its own and leaves the process's table as it found it."""
    import diff_surfel_rasterization as dsr
    monkeypatch.setattr(dsr, "_capacity", {})
    monkeypatch.setattr(dsr, "_SPECULATIVE", True)
    yield dsr


WP, WW, WH = 3000, 256, 256       # 1.25 R + 4096 at scale_modifier 1 is below R at scale_modifier 3 (asserted)


@functools.lru_cache(maxsize=None)
def wrapper_scene(O, scale_modifier):
    """Scene, identity camera and the float32 oracle's forward and gradients at one scale_modifier."""
    cam = S.to_numpy(S.make_camera(WW, WH))
    sc = S.to_numpy(S.make_scene(WP, WW, WH, 11, depth_complexity=25))
    bg = np.array([0.1, 0.2, 0.3], np.float32)
    gc, go = S.make_cotangents(WW, WH, 3)
    pre, binned, img = O.forward(sc, cam, bg, 3, scale_modifier)
    ref = O.backward(sc, cam, bg, pre, binned, img, gc.numpy(), go.numpy(), 3, scale_modifier)
    return dict(scene=sc, cam=cam, bg=bg, gc=gc, go=go, pre=pre, R=int(binned["R"]), ref=ref)


def settings(w, scale_modifier=1.0, **kw):
    from diff_surfel_rasterization import GaussianRasterizationSettings
    cam, dev = w["cam"], "cuda"
    return GaussianRasterizationSettings(
        image_height=cam["H"], image_width=cam["W"], tanfovx=cam["tanfovx"], tanfovy=cam["tanfovy"],
        bg=torch.tensor(w["bg"], device=dev), scale_modifier=scale_modifier,
        viewmatrix=torch.tensor(cam["viewmatrix"], device=dev), projmatrix=torch.tensor(cam["projmatrix"], device=dev),
        sh_degree=3, campos=torch.tensor(cam["campos"], device=dev), prefiltered=False, debug=False, **kw)


LEAVES = ("means3D", "scales", "rotations", "opacities", "shs")


def rasterize(dsr, w, rs, speculative, scene=None, grad=True, twice=False):
    """One GaussianRasterizer call (speculative launch on or off), its last_num_rendered() and, with grad, the leaf
    gradients of <cotangent, outputs> (twice: backward(retain_graph=True) then backward again; the gradients of each
    pass are returned)."""
    from diff_surfel_rasterization import GaussianRasterizer
    sc = w["scene"] if scene is None else scene
    old = dsr._SPECULATIVE
    dsr._SPECULATIVE = speculative
    try:
        leaf = {k: torch.tensor(sc[k], device="cuda", requires_grad=grad) for k in LEAVES}
        leaf["means2D"] = torch.zeros((sc["means3D"].shape[0], 3), device="cuda", requires_grad=grad)
        with torch.set_grad_enabled(grad):
            color, radii, allmap = GaussianRasterizer(rs)(means3D=leaf["means3D"], means2D=leaf["means2D"],
                                                          shs=leaf["shs"], opacities=leaf["opacities"],
                                                          scales=leaf["scales"], rotations=leaf["rotations"])
        out = dict(color=color.detach().clone(), allmap=allmap.detach().clone(), radii=radii.clone(),
                   R=dsr.last_num_rendered(), grads=[])
        if grad:
            loss = (color * w["gc"].cuda()).sum() + (allmap * w["go"].cuda()).sum()
            prev = None
            for last in ((False, True) if twice else (True,)):
                loss.backward(retain_graph=not last)
                now = {k: t.grad.detach().clone() for k, t in leaf.items()}
                out["grads"].append(now if prev is None else {k: now[k] - prev[k] for k in now})
                prev = now
        torch.cuda.synchronize()
        return out
    finally:
        dsr._SPECULATIVE = old


def assert_same_call(got, exact, what):
    assert torch.equal(bits(got["color"]), bits(exact["color"])), f"{what}: color differs from the exact-R call"
    assert torch.equal(bits(got["allmap"]), bits(exact["allmap"])), f"{what}: allmap differs from the exact-R call"
    assert torch.equal(got["radii"], exact["radii"]), f"{what}: radii differ"
    assert got["R"] == exact["R"], f"{what}: last_num_rendered() = {got['R']}, the exact call saw {exact['R']}"


def assert_grads_match_oracle(got, w, what):
    ref = w["ref"]
    for leaf, key in (("means3D", "dL_dmeans3D"), ("means2D", "dL_dmeans2D"), ("opacities", "dL_dopacity"),
                      ("shs", "dL_dshs")):
        grad_check(f"{what}: {leaf}.grad", got[leaf].cpu().numpy(), ref[key])


def key_of(w, rows=(0, 0), P=None):
    cam = w["cam"]
    return (torch.cuda.current_device(), WP if P is None else P, cam["W"], cam["H"]) + tuple(rows)


def test_repeated_calls_speculate_with_slack(oracle, cuda_lib, fresh_capacity):
    dsr, w = fresh_capacity, wrapper_scene(oracle, 1.0)
    rs = settings(w)
    exact = rasterize(dsr, w, rs, False, grad=False)
    assert exact["R"] == w["R"] and not dsr._capacity
    for i in range(3):
        got = rasterize(dsr, w, rs, True)
        assert dsr._capacity == {key_of(w): spec_cap(w["R"])}
        assert_same_call(got, exact, f"call {i + 1}")
        assert_grads_match_oracle(got["grads"][0], w, f"call {i + 1}")


def test_growth_past_the_guess_relaunches_then_shrinks(oracle, cuda_lib, fresh_capacity):
    dsr = fresh_capacity
    small, big = wrapper_scene(oracle, 1.0), wrapper_scene(oracle, 3.0)
    assert big["R"] > spec_cap(small["R"]), "scale_modifier 3 must outgrow the remembered capacity"
    key = key_of(small)
    for w, sm, cap_before in ((small, 1.0, None), (big, 3.0, spec_cap(small["R"])), (small, 1.0, spec_cap(big["R"]))):
        rs = settings(w, sm)
        exact = rasterize(dsr, w, rs, False, grad=False)
        assert exact["R"] == w["R"]
        assert dsr._capacity.get(key) == cap_before
        got = rasterize(dsr, w, rs, True)
        assert_same_call(got, exact, f"scale_modifier {sm}")
        assert_grads_match_oracle(got["grads"][0], w, f"scale_modifier {sm}")
        # a re-launch replaces the entry; a call with slack leaves it alone
        relaunched = cap_before is None or w["R"] > cap_before
        assert dsr._capacity[key] == (spec_cap(w["R"]) if relaunched else cap_before)
    assert dsr._capacity[key] == spec_cap(big["R"])


def test_backward_twice_after_relaunch(oracle, cuda_lib, fresh_capacity):
    """backward(retain_graph=True) then backward again: the first pass consumes the gradient buffers the forward
    allocated, the second allocates its own; both are the same gradient."""
    dsr = fresh_capacity
    small, big = wrapper_scene(oracle, 1.0), wrapper_scene(oracle, 3.0)
    rasterize(dsr, small, settings(small, 1.0), True, grad=False)
    rs = settings(big, 3.0)
    exact = rasterize(dsr, big, rs, False, grad=False)
    got = rasterize(dsr, big, rs, True, twice=True)
    assert dsr._capacity[key_of(big)] == spec_cap(big["R"])
    assert_same_call(got, exact, "re-launched forward")
    for i, g in enumerate(got["grads"]):
        assert_grads_match_oracle(g, big, f"backward pass {i + 1}")


def test_culled_step_after_remembered_capacity(oracle, cuda_lib, fresh_capacity):
    dsr, w = fresh_capacity, wrapper_scene(oracle, 1.0)
    rs = settings(w)
    rasterize(dsr, w, rs, True, grad=False)
    cap = dsr._capacity[key_of(w)]
    culled = {k: v.copy() for k, v in w["scene"].items()}
    culled["means3D"][:, 2] = -1.0 - np.abs(culled["means3D"][:, 2])      # every splat behind the camera
    exact = rasterize(dsr, w, rs, False, scene=culled)
    got = rasterize(dsr, w, rs, True, scene=culled)
    assert dsr._capacity[key_of(w)] == cap
    assert got["R"] == 0 and int(got["radii"].abs().max()) == 0
    assert_same_call(got, exact, "all culled")
    bgt = torch.tensor(w["bg"], device="cuda").view(3, 1, 1).expand_as(got["color"])
    assert torch.equal(got["color"], bgt) and bool((got["allmap"] == 0).all())
    for k, g in got["grads"][0].items():
        assert bool((g == 0).all()), f"{k}.grad of an all-culled step is not zero"


@pytest.mark.parametrize("replicas", [False, True])
def test_band_into_caller_buffers_through_relaunch(oracle, cuda_lib, fresh_capacity, replicas):
    """A tile band rendered into a padded caller-owned frame (plane stride > H*W) or, with replicas, into two other
    local frames: the clamped launch writes the band first, the re-launch must leave exactly the exact call's
    band, and rows outside the band stay at the sentinel."""
    dsr = fresh_capacity
    small, big = wrapper_scene(oracle, 1.0), wrapper_scene(oracle, 3.0)
    H, W = WH, WW
    band = (2, 11)

    def frames(n):
        return [torch.full((10, H + 7, W), SENTINEL, device="cuda") for _ in range(n)]

    def call(w, sm, speculative):
        local, a, b = frames(3)
        kw = dict(tile_rows=band, out_buffers=(local[:3, :H], local[3:, :H]))
        if replicas:
            kw["out_replicas"] = (a.data_ptr(), b.data_ptr())
        res = rasterize(dsr, w, settings(w, sm, **kw), speculative, grad=False)
        return res, local, a, b

    key = key_of(small, band)
    call(small, 1.0, True)
    assert dsr._capacity[key] == spec_cap(call(small, 1.0, False)[0]["R"])
    ex, ex_local, ex_a, _ = call(big, 3.0, False)
    assert ex["R"] > dsr._capacity[key], "the band must outgrow the remembered capacity"
    got, local, a, b = call(big, 3.0, True)
    assert got["R"] == ex["R"] and torch.equal(got["radii"], ex["radii"])
    assert dsr._capacity[key] == spec_cap(ex["R"])
    rows = torch.zeros(H + 7, dtype=torch.bool, device="cuda")
    rows[band[0] * 16:min(H, band[1] * 16)] = True
    targets = ((a, ex_a), (b, ex_a)) if replicas else ((local, ex_local),)
    for frame, ref in targets:
        assert torch.equal(bits(frame), bits(ref)), "the band differs from the exact call"
        assert bool((frame[:, ~rows] == SENTINEL).all()), "rows outside the band were written"
    if replicas:
        assert bool((local == SENTINEL).all()), "replica mode must not write the local out_buffers"


def test_radix_sort_never_speculates(oracle, cuda_lib, fresh_capacity):
    dsr, w = fresh_capacity, wrapper_scene(oracle, 1.0)
    rs = settings(w)
    before = "bucket" if cuda_lib.surfel_accepts_capacity() else "radix"
    assert cuda_lib.surfel_set_variant(b"sort", b"radix") == 0
    try:
        assert cuda_lib.surfel_accepts_capacity() == 0
        exact = rasterize(dsr, w, rs, False, grad=False)
        for _ in range(2):
            got = rasterize(dsr, w, rs, True, grad=False)
            assert_same_call(got, exact, "radix sort")
        assert not dsr._capacity
    finally:
        assert cuda_lib.surfel_set_variant(b"sort", before.encode()) == 0


def test_capacity_cache_bookkeeping(oracle, cuda_lib, fresh_capacity):
    """64 entries at most, the oldest evicted first; a re-launch replaces its key's entry with 1.25 R + 4096 and
    makes it the newest."""
    dsr, w = fresh_capacity, wrapper_scene(oracle, 1.0)
    rs = settings(w)
    sizes = range(1, 66)
    for P in sizes:
        part = {k: v[:P] for k, v in w["scene"].items()}
        rasterize(dsr, w, rs, True, scene=part, grad=False)
    assert len(dsr._capacity) == 64
    assert key_of(w, P=1) not in dsr._capacity
    assert list(dsr._capacity) == [key_of(w, P=P) for P in sizes[1:]]
    P = 40
    part = {k: v[:P] for k, v in w["scene"].items()}
    exact = rasterize(dsr, w, rs, False, scene=part, grad=False)
    assert exact["R"] > 1
    assert dsr._capacity[key_of(w, P=P)] == spec_cap(exact["R"])
    dsr._capacity[key_of(w, P=P)] = 1                    # a guess far too small: clamped launch, then re-launch
    got = rasterize(dsr, w, rs, True, scene=part, grad=False)
    assert_same_call(got, exact, "re-launch from a one-slot guess")
    assert len(dsr._capacity) == 64
    assert dsr._capacity[key_of(w, P=P)] == spec_cap(exact["R"])
    assert list(dsr._capacity)[-1] == key_of(w, P=P)
