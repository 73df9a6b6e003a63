"""simple_knn.distCUDA2 on the GPU: bit for bit against the certified CPU restatement (tests/knn_oracle.py), the
Python API's contract, the reference's call site (tests/golden/ref_init_knn.npz) and uninitialised scratch."""
import os

import numpy as np
import pytest
import torch

import knn_oracle as KO
import knn_scenes as KS

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32
BOX = 32            # kBox of csrc/knn.cu: points per level-0 box, the boundary the P list straddles


@pytest.fixture(scope="module")
def dev(cuda_lib):
    return torch.device("cuda:0")


def dist(points_np, dev):
    from simple_knn._C import distCUDA2
    out = distCUDA2(torch.from_numpy(np.ascontiguousarray(points_np, F32)).to(dev))
    assert out.dtype == torch.float32 and out.device == dev and out.shape == (len(points_np),)
    return out.cpu().numpy()


def assert_same(got, want):
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    bad = np.nonzero(got[ok].view(np.uint32) != want[ok].view(np.uint32))[0]
    assert bad.size == 0, f"{bad.size} rows differ, e.g. {got[ok][bad[:5]]} vs {want[ok][bad[:5]]}"


CLOUDS = {
    "uniform_100k": lambda: KS.uniform(100_000, 1),
    "colmap_like_300k": lambda: KS.colmap_like(300_000, 2),
    "uniform_4M": lambda: KS.uniform(4_000_000, 3),
    "plane_200k": lambda: KS.plane(200_000, 4),
    "line_100k": lambda: KS.line(100_000, 5),
    "lattice_40": lambda: KS.lattice(40),
    "duplicate_groups": lambda: KS.duplicate_groups([2] * 3000 + [3] * 2000 + [4] * 1000 + [500] * 20, 6),
    "10k_copies_in_200k": lambda: np.concatenate([KS.uniform(190_000, 7), KS.duplicate_groups([10_000], 7)]),
    "duplicated_300k": lambda: KS.duplicated(300_000, 8),
    "large_offset_100k": lambda: KS.large_offset(100_000, 9),
    "nonfinite_100k": lambda: KS.with_nonfinite(100_000, 10),
    "all_nonfinite": lambda: np.full((70, 3), np.nan, F32),
    "shell": lambda: KS.sphere_shell(40, 11),
}


@pytest.mark.parametrize("name", list(CLOUDS))
def test_bit_exact_against_certified_restatement(dev, name):
    pts = CLOUDS[name]()
    assert_same(dist(pts, dev), KO.mean_sq_dist(pts))


@pytest.mark.parametrize("P", [0, 1, 2, 3, 4, 5, BOX - 1, BOX, BOX + 1, 2 * BOX * BOX + 1, 65_537])
def test_bit_exact_small_and_box_boundary_counts(dev, P):
    pts = KS.uniform(P, 100 + P)
    assert_same(dist(pts, dev), KO.mean_sq_dist(pts))


def test_two_calls_identical(dev):
    from simple_knn._C import distCUDA2
    x = torch.from_numpy(KS.colmap_like(200_000, 12)).to(dev)
    a, b = distCUDA2(x), distCUDA2(x)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_non_contiguous_input(dev):
    from simple_knn._C import distCUDA2
    base = KS.uniform(50_000, 13)
    x4 = torch.cat([torch.from_numpy(base), torch.randn(50_000, 1)], 1).to(dev)
    view = x4[:, :3]
    assert not view.is_contiguous()
    assert_same(distCUDA2(view).cpu().numpy(), KO.mean_sq_dist(base))


def test_rejected_inputs(dev):
    from simple_knn._C import distCUDA2
    with pytest.raises(RuntimeError, match="float32"):
        distCUDA2(torch.zeros(8, 3, dtype=torch.float64, device=dev))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        distCUDA2(torch.zeros(8, 3))
    with pytest.raises(RuntimeError, match="shape"):
        distCUDA2(torch.zeros(8, 2, device=dev))
    with pytest.raises(RuntimeError, match="shape"):
        distCUDA2(torch.zeros(8, 3, 1, device=dev))


def test_side_stream_without_synchronisation(dev):
    """Inputs made on a side stream, the call on that stream: ordered by the stream alone.  A sleep queued ahead
    of the call is still running when the call returns, so the wrapper did not synchronise."""
    from simple_knn._C import distCUDA2
    side = torch.cuda.Stream(dev)
    g = torch.Generator(device=dev).manual_seed(14)
    with torch.cuda.stream(side):                                  # load the library, cache blocks of these sizes
        distCUDA2(torch.rand(300_000, 3, device=dev, generator=g)) * 1.0
    side.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(500_000_000)
        x = torch.rand(300_000, 3, device=dev, generator=g) * 2.6 - 1.3
        out = distCUDA2(x)
        running = not side.query()
        y = out * 1.0
    assert running, "distCUDA2 waited for the stream"
    side.synchronize()
    assert_same(y.cpu().numpy(), KO.mean_sq_dist(x.cpu().numpy()))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_second_device():
    from simple_knn._C import distCUDA2
    d1 = torch.device("cuda:1")
    pts = KS.colmap_like(100_000, 15)
    out = distCUDA2(torch.from_numpy(pts).to(d1))
    assert out.device == d1
    assert_same(out.cpu().numpy(), KO.mean_sq_dist(pts))


def test_golden_call_site(dev):
    """The stored input of the reference's create_from_pcd gives the stored distances, and the reference's two
    lines (gaussian_model.py:134-135) applied to the result give the stored _scaling: bit for bit with torch's
    CPU log / sqrt (what the golden run used), within 1 ulp with its CUDA ones (not correctly rounded)."""
    from simple_knn._C import distCUDA2
    g = np.load(os.path.join(HERE, "golden", "ref_init_knn.npz"))
    d = distCUDA2(torch.from_numpy(g["received"]).float().cuda())
    assert_same(d.cpu().numpy(), g["dist2"])
    for dist2 in (torch.clamp_min(d.cpu(), 0.0000001), torch.clamp_min(d, 0.0000001)):
        scales = torch.log(torch.sqrt(dist2))[..., None].repeat(1, 2)
        got = scales.cpu().numpy().view(np.int32).astype(np.int64)
        ulps = np.abs(got - g["scaling"].view(np.int32).astype(np.int64)).max()
        assert ulps <= (0 if dist2.device.type == "cpu" else 1), ulps


def test_poisoned_workspace(dev, cuda_lib):
    """Scratch filled with 0xFF bytes gives the same result: nothing relies on zeroed workspace."""
    from diff_surfel_rasterization import _cabi
    pts = np.concatenate([KS.colmap_like(120_000, 16), KS.with_nonfinite(1000, 16)])
    x = torch.from_numpy(pts).to(dev)
    n = cuda_lib.surfel_knn_workspace_bytes(len(pts))
    ws = torch.full((n,), 0xFF, dtype=torch.uint8, device=dev)
    out = torch.full((len(pts),), 7.0, device=dev)
    _cabi.check(cuda_lib.surfel_knn_mean_sq_dist(len(pts), x.data_ptr(), out.data_ptr(), ws.data_ptr(), n,
                                                 torch.cuda.current_stream(dev).cuda_stream))
    assert_same(out.cpu().numpy(), KO.mean_sq_dist(pts))
