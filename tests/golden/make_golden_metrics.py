"""Records what THE REFERENCE'S OWN metrics.py computes per view (ssim of utils/loss_utils.py, psnr of
utils/image_utils.py, lpips(render, gt, net_type='vgg') of lpipsPyTorch), for diff_surfel_rasterization.metrics
(DESIGN.md §7o).

metrics.py is loaded with runpy (not as __main__) and its evaluate() runs unmodified on a temporary
<scene>/test/<method>/{renders,gt} tree of PNGs written with PIL.  evaluate() swallows every exception, so the
generator checks that it wrote results.json and per_view.json.  torch, torchvision and PIL are real and run on the
CPU.  What is stubbed:
  * torch.Tensor.cuda is the identity (the tensors stay on the CPU);
  * matplotlib (utils/image_utils.py imports pyplot, and matplotlib is not installed) is an empty module;
  * tqdm passes its iterable through;
  * torchvision.models.vgg16 returns the real architecture with the seeded conv weights of tests/metrics_ref.py.
    It reseeds on every construction, because lpips() builds a new LPIPS per image;
  * torch.hub.load_state_dict_from_url serves the seeded lin weights under LPIPS's own key names.
Then the reference's LPIPS module itself is run on the small cases to record its five taps' (normalized)
features, and in float64 (.double() on the module and both images) for the float64 value.

Writes tests/golden/ref_metrics.npz.  Re-running gives the same file bit for bit.

Usage:  python tests/golden/make_golden_metrics.py
"""
import io
import json
import os
import runpy
import sys
import tempfile
import types
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
REF = "/root/reference"
OUT = os.path.join(HERE, "ref_metrics.npz")
FEATURE_CASES = ("min_16x16", "odd_35x17")     # the five taps' features are recorded for these (the file stays small)

import metrics_ref as R  # noqa: E402


def cases():
    """name -> (render uint8 (H,W,3|4), gt uint8 (H,W,3)); seeded, written as PNGs."""
    rng = np.random.default_rng(R.SEED)
    out = {}

    def smooth(h, w):
        lo = rng.random((h // 4 + 2, w // 4 + 2, 3))
        ys, xs = np.linspace(0, lo.shape[0] - 1, h), np.linspace(0, lo.shape[1] - 1, w)
        y0, x0 = np.floor(ys).astype(int), np.floor(xs).astype(int)
        y1, x1 = np.minimum(y0 + 1, lo.shape[0] - 1), np.minimum(x0 + 1, lo.shape[1] - 1)
        fy, fx = (ys - y0)[:, None, None], (xs - x0)[None, :, None]
        v = (lo[y0][:, x0] * (1 - fy) * (1 - fx) + lo[y1][:, x0] * fy * (1 - fx) + lo[y0][:, x1] * (1 - fy) * fx
             + lo[y1][:, x1] * fy * fx)
        return v

    def q(v):
        return np.clip(np.round(v * 255), 0, 255).astype(np.uint8)

    for name, (h, w, s) in {"even_32x48": (32, 48, 0.05), "odd_37x53": (37, 53, 0.1), "odd_35x17": (35, 17, 0.03),
                            "pool_31x63": (31, 63, 0.08), "min_16x16": (16, 16, 0.05), "min_16x23": (16, 23, 0.1)}.items():
        gt = smooth(h, w)
        out[name] = (q(gt + s * rng.standard_normal(gt.shape)), q(gt))
    gt = smooth(24, 20)
    rgba = np.concatenate([q(gt + 0.05 * rng.standard_normal(gt.shape)), rng.integers(0, 256, (24, 20, 1), np.uint8)], 2)
    out["rgba_24x20"] = (rgba, q(gt))
    img = q(smooth(20, 18))
    out["identical_20x18"] = (img, img.copy())
    gt = smooth(24, 24)
    out["black_24x24"] = (np.zeros((24, 24, 3), np.uint8), q(gt))
    return out


def install_stubs():
    import torch
    import torchvision

    torch.Tensor.cuda = lambda self, *a, **k: self
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, mpl.pyplot
    tq = types.ModuleType("tqdm")
    tq.tqdm = lambda it, *a, **k: it
    sys.modules["tqdm"] = tq
    real_vgg16 = torchvision.models.vgg16

    def vgg16(weights=None, **kw):
        m = real_vgg16(weights=None)
        sd = R.vgg_weights()                       # reseeded on every construction
        m.features.load_state_dict({k[len("features."):]: v for k, v in sd.items()})
        return m

    torchvision.models.vgg16 = vgg16

    def load_state_dict_from_url(url, **kw):
        assert url.endswith("/vgg.pth"), url
        return R.lin_weights()

    torch.hub.load_state_dict_from_url = load_state_dict_from_url


def main():
    import torch
    from PIL import Image

    torch.use_deterministic_algorithms(True)
    install_stubs()
    sys.path.insert(0, REF)
    ns = runpy.run_path(os.path.join(REF, "metrics.py"), run_name="metrics_golden")
    from lpipsPyTorch.modules.lpips import LPIPS

    cs = cases()
    rec = {"names": np.array(sorted(cs)), "seed": np.int64(R.SEED), "min_side": np.int64(R.MIN_SIDE),
           "weights_sha256": np.array(R.weights_sha256(R.vgg_weights(), R.lin_weights()))}
    with tempfile.TemporaryDirectory() as tmp:
        scene = os.path.join(tmp, "scene")
        mdir = os.path.join(scene, "test", "ours_30000")
        for sub in ("renders", "gt"):
            os.makedirs(os.path.join(mdir, sub))
        for name, (r, g) in cs.items():
            Image.fromarray(r).save(os.path.join(mdir, "renders", name + ".png"))
            Image.fromarray(g).save(os.path.join(mdir, "gt", name + ".png"))
        ns["evaluate"]([scene])
        for f in ("results.json", "per_view.json"):
            if not os.path.exists(os.path.join(scene, f)):
                raise RuntimeError(f"metrics.py evaluate() wrote no {f}: it failed (it swallows the exception)")
        with open(os.path.join(scene, "per_view.json")) as fp:
            per_view = json.load(fp)["ours_30000"]
        from pathlib import Path
        renders, gts, names = ns["readImages"](Path(mdir) / "renders", Path(mdir) / "gt")
        imgs = {n[:-4]: (r, g) for r, g, n in zip(renders, gts, names)}
    for name in sorted(cs):
        r, g = imgs[name]
        rec[f"{name}/render"], rec[f"{name}/gt"] = r.numpy(), g.numpy()
        for key, m in (("ssim", "SSIM"), ("psnr", "PSNR"), ("lpips", "LPIPS")):
            rec[f"{name}/{key}"] = np.float32(per_view[m][name + ".png"])
        crit = LPIPS("vgg", "0.1")
        with torch.no_grad():
            if name in FEATURE_CASES:
                for i, f in enumerate(crit.net(r)):
                    rec[f"{name}/feat{i}"] = f.numpy()
            crit64 = crit.double()
            rec[f"{name}/lpips_f64"] = np.float64(crit64(r.double(), g.double()).item())
    # the smallest side the reference accepts: 16 runs, 15 leaves conv5 an empty image
    crit = LPIPS("vgg", "0.1")
    x = torch.rand((1, 3, 15, 40), generator=torch.Generator().manual_seed(0))
    try:
        with torch.no_grad():
            crit(x, x)
        rec["rejects_15"] = np.bool_(False)
    except RuntimeError:
        rec["rejects_15"] = np.bool_(True)
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED) as z:     # fixed timestamps: the same bytes every run
        for k in sorted(rec):
            b = io.BytesIO()
            np.save(b, rec[k], allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, b.getvalue())
    with open(OUT, "wb") as f:
        f.write(buf.getvalue())
    print(f"wrote {OUT}: {len(cs)} cases, {os.path.getsize(OUT)} bytes")
    for name in sorted(cs):
        print(f"  {name:16s} ssim {rec[name + '/ssim']:.6f} psnr {rec[name + '/psnr']:.4f} "
              f"lpips {rec[name + '/lpips']:.6f} f64 {rec[name + '/lpips_f64']:.6f}")


if __name__ == "__main__":
    main()
