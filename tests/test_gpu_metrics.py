"""The evaluation script's 8-bit PSNR and SSIM on the GPU (f2b_image_metrics, csrc/metrics.cu; eval.ImageMetrics and the
"psnr_8bit" / "ssim" outputs of eval.TestImages) against the reference script's own values (tests/golden/ref_eval_metrics.npz)
and the float64 restatement (tests/image_metrics_oracle.py): the SSE exactly, so the PSNR to the last bit, and the SSIM to 1e-9."""
import os

import numpy as np
import pytest
import torch

import image_metrics_oracle as IM

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
METRICS = os.path.join(ROOT, "tests", "golden", "ref_eval_metrics.npz")


def from_u8(a):
    """A uint8 image as the reference loads it (u8 / 255.f on the CPU), on the device."""
    return (torch.from_numpy(a).to(torch.float32) / 255.).cuda()


def device_sums(pred, gt):
    from f2nerf_b200.eval import _image_metrics
    sse, ssim_sum = _image_metrics(pred, gt)
    return int(sse.item()), ssim_sum.item()


def test_image_metrics_match_reference_fixture():
    from f2nerf_b200 import ImageMetrics
    d = dict(np.load(METRICS))
    for n in (str(n) for n in d["names"]):
        gt, pred = d[f"{n}_gt"], d[f"{n}_pred"]
        m = ImageMetrics(from_u8(pred), from_u8(gt))
        assert device_sums(from_u8(pred), from_u8(gt))[0] == IM.sse(pred, gt), n
        assert m["psnr_8bit"] == float(d[f"{n}_psnr"]) == IM.psnr(pred, gt), n
        assert abs(m["ssim"] - float(d[f"{n}_ssim"])) <= 1e-9, (n, m["ssim"], float(d[f"{n}_ssim"]))
        assert abs(m["ssim"] - IM.ssim(pred, gt)) <= 1e-9, n
    assert ImageMetrics(from_u8(d["identical_pred"]), from_u8(d["identical_gt"]))["psnr_8bit"] == float("inf")


def seeded_pair(h, w, seed):
    """A smooth ground truth off the 1/255 grid with noise, and a prediction near it that leaves [0, 1] in places."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    base = torch.stack([0.5 + 0.4 * torch.sin(xx / 9.) * torch.cos(yy / 13.), (xx + yy) / (h + w), (xx > w / 3).float()], -1)
    gt = (base + 0.03 * torch.randn((h, w, 3), generator=g)).clip(0., 1.)
    pred = gt + 0.05 * torch.randn((h, w, 3), generator=g)
    return pred, gt


# 32 x 16 outputs per tile: 42 x 26 is one tile exactly, 43 x 27 one past; 1080 x 1920 has more tiles than the grid has CTAs
@pytest.mark.parametrize("h,w", [(11, 11), (26, 42), (27, 43), (11, 300), (301, 11), (37, 53), (129, 257), (540, 960), (1080, 1920)])
def test_image_metrics_match_restatement(h, w):
    from f2nerf_b200 import ImageMetrics
    pred, gt = seeded_pair(h, w, seed=h * 7919 + w)
    assert float(pred.min()) < 0. and float(pred.max()) > 1.
    p8, g8 = IM.pred_to_u8(pred.numpy()), IM.gt_to_u8(gt.numpy())
    sse, ssim_sum = device_sums(pred.cuda(), gt.cuda())
    assert sse == IM.sse(p8, g8)
    assert abs(ssim_sum / ((h - 10) * (w - 10) * 3) - IM.ssim(p8, g8)) <= 1e-9
    m = ImageMetrics(pred.cuda(), gt.cuda())
    assert m["psnr_8bit"] == IM.psnr(p8, g8)
    assert abs(m["ssim"] - IM.ssim(p8, g8)) <= 1e-9


def test_image_metrics_identical_images_and_determinism():
    from f2nerf_b200 import ImageMetrics
    img = from_u8(np.random.default_rng(3).integers(0, 256, (1080, 1920, 3), dtype=np.uint8))   # the same bytes by both rules
    m = ImageMetrics(img, img)
    assert m["psnr_8bit"] == float("inf") and abs(m["ssim"] - 1.) <= 1e-12
    pred, gt = seeded_pair(1080, 1920, seed=3)
    runs = [device_sums(pred.cuda(), gt.cuda()) for _ in range(2)]
    assert runs[0][0] == runs[1][0]
    assert np.float64(runs[0][1]).view(np.uint64) == np.float64(runs[1][1]).view(np.uint64)


def test_image_metrics_refuses_bad_inputs():
    from f2nerf_b200 import ImageMetrics
    from f2nerf_b200._lib import F2BError
    for h, w in ((10, 40), (40, 10), (10, 10)):
        x = torch.rand((h, w, 3), device="cuda")
        with pytest.raises(F2BError, match="smaller than"):
            ImageMetrics(x, x)
    x = torch.rand((20, 20, 3), device="cuda")
    for a, b in ((x, x[:, :19]), (x[..., :1], x[..., :1]), (x.cpu(), x.cpu()), (x.reshape(-1), x.reshape(-1))):
        with pytest.raises(ValueError):
            ImageMetrics(a, b)


def test_test_images_scores_match_restatement():
    """TestImages' "psnr_8bit" / "ssim" on the ngp_fox scene (3 views of 960 x 540, ground truth off the 1/255 grid) == the
    restatement applied to the same quantised colours and ground truth; a second run gives the same bits."""
    from f2nerf_b200 import ImageMetrics, TestImages
    from test_gpu_eval import ngp_fox
    gdp, renderer, gen = ngp_fox()
    res = TestImages(renderer, gen)
    again = TestImages(renderer, gen)
    assert sorted(res["psnr_8bit"]) == sorted(res["ssim"]) == gen.test_set_
    for k, idx in enumerate(gen.test_set_):
        q, gt = res["colors"][k], gen.image_tensors_[idx]
        g = gt.cpu().numpy()
        assert np.any(IM.gt_to_u8(g) != np.trunc(g * np.float32(255.)))          # the rint rule has work to do
        p8, g8 = IM.pred_to_u8(q.cpu().numpy()), IM.gt_to_u8(g)
        assert res["psnr_8bit"][idx] == IM.psnr(p8, g8)
        assert abs(res["ssim"][idx] - IM.ssim(p8, g8)) <= 1e-9
        m = ImageMetrics(q, gt)
        assert m["psnr_8bit"] == res["psnr_8bit"][idx] and m["ssim"] == res["ssim"][idx]
        for key in ("psnr", "psnr_8bit", "ssim"):
            assert np.float64(again[key][idx]).view(np.uint64) == np.float64(res[key][idx]).view(np.uint64), key
    n = len(gen.test_set_)
    assert res["mean_psnr_8bit"] == sum(res["psnr_8bit"].values()) / n
    assert res["mean_ssim"] == sum(res["ssim"].values()) / n
