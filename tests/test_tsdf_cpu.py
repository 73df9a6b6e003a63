"""The unbounded TSDF field without a device (DESIGN.md §7i): the float64 evaluation against the reference's stored
outputs, the float32 emulation of csrc/tsdf.cu against the bounds, each quirk on a hand-built case, and the C ABI's
argument checks."""
import ctypes
import os

import numpy as np
import pytest

import tsdf_ref as TR
import tsdf_scenes as TS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_tsdf.npz")
F = np.float32


def golden():
    g = np.load(GOLDEN)
    frames = [(g[f"proj{f}"], g[f"depth{f}"][0], g[f"rgb{f}"]) for f in range(int(g["n_frames"]))]
    return g, frames, (g["center"], float(g["radius"]), 5 * float(g["voxel_size"]))


@pytest.mark.parametrize("colour", [False, True])
def test_float64_evaluation_reproduces_the_reference(colour):
    g, frames, args = golden()
    pts, ref = (g["colour_points"], g["ref_rgb"]) if colour else (g["points"], g["ref_tsdf"])
    value, bound, flagged = TR.evaluate64(pts, frames, *args, colour=colour)
    assert flagged.mean() < 1e-3
    assert len(TR.check_within(ref, value, bound, flagged, factor=1.0)) == 0
    if not colour:
        assert np.all(ref[flagged] >= -1) and np.all(ref[flagged] <= 1)
        # the same unobserved (-1) samples, and no NaN: a NaN tap rejects its frame
        assert np.array_equal(ref[~flagged] == -1, value[~flagged] == -1)
        assert not np.isnan(ref).any() and (ref != -1).sum() > 500
    else:
        assert (ref != 0).any(1).sum() > 500


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("colour", [False, True])
def test_emulation_stays_inside_the_bounds(seed, colour):
    rng = np.random.default_rng(seed)
    sizes = [(int(rng.integers(1, 70)), int(rng.integers(1, 60))) for _ in range(6)] + [(1, 9), (9, 1), (1, 1)]
    views = TS.analytic_views(sizes, seed)
    frames = TS.frames_of(views)
    radius, center = 2.7 + seed * 0.1, np.array([0.05, -0.1, 0.02], F)
    if colour:
        pts = np.concatenate([rng.uniform(-2, 2, (6000, 3)), TS.sphere_surface_points(2000, rng, center, radius)[1]])
    else:
        pts = np.concatenate([rng.uniform(-1.9, 1.9, (8000, 3)), TS.special_points(1.9),
                              TS.sphere_surface_points(2000, rng, center, radius)[0]])
    pts = pts.astype(F)
    value, bound, flagged = TR.evaluate64(pts, frames, center, radius, 5 * radius * 2 / 1024, colour=colour)
    got = TR.emulate(pts, frames, center, radius, 5 * radius * 2 / 1024, colour=colour)
    assert flagged.mean() < 1e-3
    assert len(TR.check_within(got, value, bound, flagged, factor=1.0)) == 0
    observed = (got != 0).any(1) if colour else got != -1
    assert observed.sum() > 200


# ---- the quirks, each on a hand-built case -------------------------------------------------------------------------

def _identity_view(W=5, H=4, depth=2.0):
    """A camera at the origin looking down +z with tan(fov/2) = 1: pix = (x/z, y/z), w = z.  The field-mode cases
    below use radius 4 and points inside the unit ball, so a sample y is the world point 4 y."""
    M = np.zeros((4, 4), F)
    M[0, 0] = M[1, 1] = M[2, 3] = 1
    return M, np.full((H, W), depth, F), np.stack([np.full((H, W), c, F) for c in (0.2, 0.4, 0.6)])


def test_unobserved_sample_is_minus_one_and_first_observation_averages_with_it():
    M, d, c = _identity_view(depth=2.0)
    pts = np.array([[0, 0, 1.5], [0, 0, -1.0]], F)
    t = TR.emulate(pts / 4, [(M, d, c)], [0, 0, 0], 4.0, 1.0)
    assert t[1] == -1
    assert t[0] == F((F(-1) * 1 + F(0.5)) / 2)                     # s = clamp(0.5 / 1) averaged with -1
    rgb = TR.emulate(pts, [(M, d, c)], [0, 0, 0], 1.0, 1.0, colour=True)
    assert np.array_equal(rgb[0], (c[:, 0, 0] / 2).astype(F)) and np.all(rgb[1] == 0)


def test_fold_depends_on_frame_order():
    # the mean of the same observations, rounded at every step: some orders differ in the last bit
    M, _, c = _identity_view()
    pts = np.array([[0, 0, 1.5]], F) / 4
    differ = 0
    rng = np.random.default_rng(0)
    for _ in range(20):
        frames = [(M, np.full((4, 5), v, F), c) for v in rng.uniform(1.2, 2.4, 6)]
        differ += TR.emulate(pts, frames, [0, 0, 0], 4.0, 1.0)[0] != TR.emulate(pts, frames[::-1], [0, 0, 0], 4.0, 1.0)[0]
    assert differ > 0


def test_uncontract_edges():
    with np.errstate(all="ignore"):
        X, Y, Z, _ = TR.world_and_trunc32(np.array([[2, 0, 0], [1.9, 1.9, 1.9], [1, 0, 0]], F), [0, 0, 0], 1.0, 1.0,
                                          False)
    assert np.isinf(X[0]) and np.isnan(Y[0])                     # |y| = 2: inf / NaN, never observed
    assert np.allclose([X[1], Y[1], Z[1]], -0.447, atol=1e-3)     # the corner lands on the opposite side
    assert (X[2], Y[2], Z[2]) == (1, 0, 0)                        # |y| = 1 takes the contracted branch: 1/(2-1) * y
    M, d, c = _identity_view()
    assert TR.emulate(np.array([[0, 0, 2]], F), [(M, d, c)], [0, 0, 0], 1.0, 1.0)[0] == -1


def test_adaptive_truncation():
    t0 = 5 * 0.01
    pts = np.array([[0.5, 0, 0], [1.5, 0, 0], [0, 1.95, 0], [0, 0, 3.0]], F)
    _, _, _, tr = TR.world_and_trunc32(pts, [0, 0, 0], 1.0, t0, False)
    assert tr[0] == F(t0)
    assert tr[1] == F(t0) * (F(1) / (F(2) - F(1.5)))
    assert tr[2] == tr[3] == F(t0) * (F(1) / (F(2) - F(1.9)))     # clamped at 1.9
    _, _, _, trc = TR.world_and_trunc32(pts, [0, 0, 0], 1.0, t0, True)
    assert np.all(trc == F(t0))                                    # colour pass: the plain scalar


def test_mask_and_clamp():
    M, d, c = _identity_view(depth=2.0)
    one = lambda p, trunc=0.25: TR.emulate(np.array([p], F) / 4, [(M, d, c)], [0, 0, 0], 4.0, trunc)[0]
    assert one([0, 0, 0.5]) == F(0)                                # far in front: sdf / trunc clamps to +1
    assert one([0, 0, 0.5], trunc=1e3) != 0                        # not clamped
    assert one([0.99, 0, 0.5]) == -1                               # pix = 1.98: outside
    assert one([0, 0, 2.2]) != -1                                  # behind the surface, within trunc
    assert one([0, 0, 2.2], trunc=0.1) == -1                       # beyond -trunc
    assert one([0, 0, -0.5]) == -1                                 # z < 0


def test_nan_tap_at_zero_weight_rejects_and_empty_pixels_give_minus_z():
    H, W = 3, 5
    M, _, c = _identity_view(W, H)
    # pix (0, 0) is pixel (row 1, column 2) exactly; its east neighbour is NaN and has weight 0
    d = np.full((H, W), 3.0, F)
    d2 = d.copy()
    d2[1, 3] = np.nan
    p = np.array([[0, 0, 1.5]], F) / 4
    assert TR.emulate(p, [(M, d2, c)], [0, 0, 0], 4.0, 10.0)[0] == -1
    assert TR.emulate(p, [(M, d, c)], [0, 0, 0], 4.0, 10.0)[0] != -1
    t = TR.emulate(p, [(M, np.zeros((H, W), F), c)], [0, 0, 0], 4.0, 10.0)[0]
    assert t == F((F(-1) + F(-1.5) / F(10)) / F(2))                # an empty pixel: sdf = 0 - z


def test_bilinear_border_taps():
    m = np.arange(12, dtype=F).reshape(3, 4)
    v = TR._bilinear32(m, np.array([1 - 2 ** -23, -1 + 2 ** -23, 0.0], F), np.array([0.0, 0.0, 1 - 2 ** -23], F))
    assert abs(v[0] - 7) < 1e-5 and abs(v[1] - 4) < 1e-5 and abs(v[2] - 9.5) < 1e-5


# ---- the entry point and the C ABI without a device ----------------------------------------------------------------

def test_python_entry_rejects_bad_arguments_without_a_device():
    import types
    import torch
    from diff_surfel_rasterization.tsdf import UnboundedTSDF
    cam = types.SimpleNamespace(full_proj_transform=torch.eye(4))
    d, c = torch.zeros(1, 4, 5), torch.zeros(3, 4, 5)
    with pytest.raises(RuntimeError, match="cameras"):
        UnboundedTSDF([d, d], [c, c], [cam], torch.zeros(3), 1.0, 0.01)
    with pytest.raises(RuntimeError, match="RGB map"):
        UnboundedTSDF([d], [torch.zeros(3, 4, 6)], [cam], torch.zeros(3), 1.0, 0.01)
    with pytest.raises(RuntimeError, match="full_proj_transform"):
        UnboundedTSDF([d], [c], [types.SimpleNamespace(full_proj_transform=torch.eye(3))], torch.zeros(3), 1.0, 0.01)
    with pytest.raises(RuntimeError, match="depth map"):
        UnboundedTSDF([torch.zeros(4, 5)], [c], [cam], torch.zeros(3), 1.0, 0.01)


def test_cabi_rejects_bad_arguments_without_a_device():
    from diff_surfel_rasterization import _cabi
    lib = _cabi.load()
    err = lambda: lib.surfel_last_error().decode()
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    center = (ctypes.c_float * 3)(0, 0, 0)
    frames = (_cabi.TsdfFrame * 2)()
    for f, fr in enumerate(frames):
        fr.height, fr.width, fr.offset = 4, 5, 20 * f
    call = lambda n=8, pts=p, V=2, fr=frames, mp=40, d=p, rgb=None, cen=center, out=p: lib.surfel_tsdf_eval(
        n, pts, V, fr, mp, d, rgb, cen, 1.0, 0.05, out, None)
    assert call(n=-1) != 0 and "negative" in err()
    assert call(V=-1) != 0 and "negative" in err()
    assert call(mp=-1) != 0 and "negative" in err()
    assert call(n=1 << 40) != 0 and "grid" in err()
    assert call(cen=None) != 0 and "center" in err()
    assert call(fr=None) != 0 and "frame table" in err()
    assert call(pts=None) != 0 and "NULL points" in err()
    assert call(out=None) != 0 and "NULL points or output" in err()
    assert call(d=None) != 0 and "depth" in err()
    assert call(mp=39) != 0 and "outside" in err()
    frames[1].offset = -1
    assert call() != 0 and "outside" in err()
    frames[1].offset, frames[1].width = 20, 0
    assert call() != 0 and "2^24" in err()
    frames[1].width, frames[1].height = 5, (1 << 24) + 1
    assert call(mp=1 << 40) != 0 and "2^24" in err()
    frames[1].height = 4
    assert call(n=0) == 0                                          # nothing to do: no launch, no device needed
    assert call(n=0, V=0, fr=None, mp=0, d=None) == 0
