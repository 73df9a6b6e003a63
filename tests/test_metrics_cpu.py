"""The restatement of metrics.py's PSNR and LPIPS-VGG (tests/metrics_ref.py) against the reference's own values
(tests/golden/ref_metrics.npz), the package's weight loading, and the C ABI's argument checks; no GPU."""
import ctypes

import numpy as np
import pytest
import torch

import metrics_ref as R

GOLDEN = __import__("os").path.join(__import__("os").path.dirname(__import__("os").path.abspath(__file__)),
                                    "golden", "ref_metrics.npz")


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def weights():
    return R.vgg_weights(), R.lin_weights()


def _names(z):
    return [str(n) for n in z["names"]]


def test_weights_regenerate(z, weights):
    assert int(z["seed"]) == R.SEED
    assert str(z["weights_sha256"]) == R.weights_sha256(*weights)


def test_golden_covers_the_cases(z):
    names = _names(z)
    shapes = [z[f"{n}/render"].shape[-2:] for n in names]
    assert int(z["min_side"]) == R.MIN_SIDE and bool(z["rejects_15"])
    assert any(min(s) == R.MIN_SIDE for s in shapes)
    assert any(h % 2 and w % 2 for h, w in shapes)
    assert any(h % 2 == 0 and w % 2 == 0 for h, w in shapes)
    assert any(n.startswith("rgba") for n in names) and any(n.startswith("black") for n in names)
    ident = [n for n in names if n.startswith("identical")]
    assert ident and all(float(z[f"{n}/lpips"]) == 0.0 and np.isinf(z[f"{n}/psnr"]) for n in ident)


def test_input_tensors(z):
    """[0,1] float32 values k/255, three channels (alpha dropped), not rescaled."""
    for n in _names(z):
        for key in ("render", "gt"):
            t = z[f"{n}/{key}"]
            assert t.dtype == np.float32 and t.shape[:2] == (1, 3)
            k = np.round(t.astype(np.float64) * 255)
            assert np.array_equal((k / 255).astype(np.float32), t) and t.min() >= 0 and t.max() <= 1
    assert z["black_24x24/render"].max() == 0.0


@pytest.mark.parametrize("name", ["black_24x24", "even_32x48", "identical_20x18", "min_16x16", "min_16x23",
                                  "odd_35x17", "odd_37x53", "pool_31x63", "rgba_24x20"])
def test_restatement_matches_reference(z, weights, name):
    x, y = torch.from_numpy(z[f"{name}/render"]), torch.from_numpy(z[f"{name}/gt"])
    v64, taps, fx, _ = R.lpips_f64(x, y, *weights)
    assert abs(v64 - float(z[f"{name}/lpips_f64"])) <= 1e-12 * max(1.0, abs(v64))
    # the reference's float32 value, within float32 noise of a 13-layer network
    assert abs(v64 - float(z[f"{name}/lpips"])) <= 1e-5 * max(abs(v64), 1e-2)
    if f"{name}/feat0" in z:
        for i, f in enumerate(fx):
            want = z[f"{name}/feat{i}"].astype(np.float64)
            got = R.normalize(f).numpy()
            assert np.abs(got - want).max() <= 1e-5
    p64 = float(R.psnr_f64(x, y)[0])
    p32 = float(z[f"{name}/psnr"])
    if np.isinf(p32):
        assert np.isinf(p64)
    else:
        assert abs(p64 - p32) <= 1e-4


def test_load_maps_keys(tmp_path, weights, monkeypatch):
    from diff_surfel_rasterization import metrics
    vgg, lin = weights
    captured = {}

    def fake_init(self, v, l, device=None):
        captured["vgg"], captured["lin"], captured["device"] = v, l, device

    monkeypatch.setattr(metrics.LPIPS, "__init__", fake_init)
    vp, lp = tmp_path / "v.pth", tmp_path / "l.pth"
    torch.save({k: v[:1].clone() for k, v in vgg.items()}, vp)
    torch.save(lin, lp)
    metrics.LPIPS.load(str(vp), str(lp), device="cuda:3")
    assert sorted(captured["vgg"]) == sorted(vgg) and captured["device"] == "cuda:3"
    assert all(torch.equal(captured["lin"][k], lin[k]) for k in lin)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    (tmp_path / "checkpoints").mkdir()
    with pytest.raises(FileNotFoundError, match="vgg16-397923af.pth"):
        metrics.LPIPS.load()
    torch.save(lin, tmp_path / "checkpoints" / "vgg16-397923af.pth")
    with pytest.raises(FileNotFoundError, match="vgg.pth"):
        metrics.LPIPS.load()
    torch.save(lin, tmp_path / "checkpoints" / "vgg.pth")
    metrics.LPIPS.load()
    assert sorted(captured["vgg"]) == sorted(lin)


def test_state_dict_checks():
    from diff_surfel_rasterization.metrics import _param
    with pytest.raises(KeyError, match="features.0.weight"):
        _param({}, "features.0.weight", (64, 3, 3, 3))
    with pytest.raises(ValueError, match="shape"):
        _param({"w": torch.zeros(2)}, "w", (3,))


def _lib():
    from diff_surfel_rasterization import _cabi
    try:
        return _cabi.load()
    except ImportError as ex:
        pytest.skip(f"library not built: {ex}")


def test_c_abi_rejects_bad_arguments():
    lib = _lib()
    p = ctypes.c_void_p(16)
    assert lib.surfel_metrics_min_side() == R.MIN_SIDE
    assert lib.surfel_metrics_partials_count(0) == 0 and lib.surfel_metrics_partials_count(3) >= 5 * 1
    host = (ctypes.c_float * (3 * 32 * 32))()
    assert lib.surfel_metrics_lpips_input(1, 3, 15, 40, p, p, p, None) != 0
    assert b"outside" in lib.surfel_last_error()
    assert lib.surfel_metrics_lpips_input(1, 3, 40, 15, p, p, p, None) != 0
    assert lib.surfel_metrics_lpips_input(2, 3, 40, 40, p, p, p, None) != 0
    assert b"batch" in lib.surfel_last_error()
    assert lib.surfel_metrics_lpips_input(1, 4, 40, 40, p, p, p, None) != 0
    assert b"channels" in lib.surfel_last_error()
    assert lib.surfel_metrics_lpips_input(1, 3, 32, 32, host, host, host, None) != 0
    assert b"device memory" in lib.surfel_last_error()
    assert lib.surfel_metrics_lpips_input(1, 3, 32, 32, None, p, p, None) != 0
    assert b"NULL" in lib.surfel_last_error()
    assert lib.surfel_metrics_psnr(1, 3 * 32 * 32, host, host, p, p, None) != 0
    assert b"device memory" in lib.surfel_last_error()
    assert lib.surfel_metrics_psnr(0, 10, p, p, p, p, None) != 0
    assert lib.surfel_metrics_conv3x3(2, 32, 32, 48, 64, p, p, p, p, None) != 0
    assert b"unsupported" in lib.surfel_last_error()
    assert lib.surfel_metrics_conv3x3(3, 32, 32, 64, 64, p, p, p, p, None) != 0
    assert lib.surfel_metrics_conv3x3(2, 32, 32, 64, 64, p, None, p, p, None) != 0
    assert lib.surfel_metrics_pack_conv(100, 64, p, p, None) != 0
    assert lib.surfel_metrics_maxpool(2, 1, 32, 64, p, p, None) != 0
    assert lib.surfel_metrics_maxpool(2, 32, 32, 6, p, p, None) != 0
    assert lib.surfel_metrics_lpips_tap(5, 32, 32, 64, p, p, p, None) != 0
    assert lib.surfel_metrics_lpips_tap(0, 32, 32, 1024, p, p, p, None) != 0
    pix = (ctypes.c_longlong * 5)(4, 4, 4, 4, 0)
    assert lib.surfel_metrics_lpips_finish(pix, p, p, None, None) != 0
    assert b"empty" in lib.surfel_last_error()


def test_python_rejects_non_cuda():
    from diff_surfel_rasterization.metrics import LPIPS, psnr, ssim
    x = torch.rand((1, 3, 32, 32))
    with pytest.raises(TypeError):
        psnr(x, x)
    with pytest.raises(TypeError):
        ssim(x, x)
    with pytest.raises(TypeError):
        LPIPS.__call__(object.__new__(LPIPS), x, x)
