"""CPU checks of the evaluation script's image metrics: the float64 restatement (tests/image_metrics_oracle.py) against the
reference's own values (tests/golden/ref_eval_metrics.npz), the 8-bit conversion rules against the reference's writer, and the
host-side pieces of eval.ImageMetrics (filter taps, PSNR formula)."""
import os

import numpy as np
import pytest
import torch

import image_metrics_oracle as IM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
METRICS = os.path.join(ROOT, "tests", "golden", "ref_eval_metrics.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(METRICS))


def test_fixture_is_small_and_complete(golden):
    assert os.path.getsize(METRICS) < 100 * 1024
    names = [str(n) for n in golden["names"]]
    shapes = {golden[f"{n}_gt"].shape[:2] for n in names}
    assert (11, 11) in shapes and any(h % 2 and w % 2 for h, w in shapes)
    for n in names:
        assert golden[f"{n}_gt"].dtype == np.uint8 and golden[f"{n}_gt"].shape == golden[f"{n}_pred"].shape
    assert np.isinf(golden["identical_psnr"]) and np.ptp(golden["constant_gt_gt"]) == 0


def test_restatement_matches_reference(golden):
    """PSNR exactly, SSIM to 1e-12 of scripts/eval.py's own rgb_ssim."""
    for n in (str(n) for n in golden["names"]):
        gt, pred = golden[f"{n}_gt"], golden[f"{n}_pred"]
        assert IM.psnr(gt, pred) == float(golden[f"{n}_psnr"]), n
        assert abs(IM.ssim(gt, pred) - float(golden[f"{n}_ssim"])) <= 1e-12, n


def quantify_then_write(x):
    """ExpRunner::TestImages' quantify (ExpRunner.cpp:360-362) then Utils::WriteImageTensor's cast (ImageIO.cpp:29), on CPU
    tensors as the reference runs them."""
    q = (x.clip(0., 1.) * 255.).to(torch.uint8).to(torch.float32) / 255.
    return (q * 255.).clip(0., 255.).to(torch.uint8)


def test_pred_rule_is_the_writer_of_quantified_colours():
    levels = torch.arange(256, dtype=torch.float32)
    np.testing.assert_array_equal(IM.pred_to_u8((levels / 255.).numpy()), np.arange(256))
    for x in (levels / 255., levels / 255. + 1e-4, (levels + 0.999) / 255., torch.linspace(-0.5, 1.5, 200001)):
        want = quantify_then_write(x).numpy()
        np.testing.assert_array_equal(IM.pred_to_u8(x.numpy()), want)
        q = (x.clip(0., 1.) * 255.).to(torch.uint8).to(torch.float32) / 255.                 # the quantised colours themselves
        np.testing.assert_array_equal(IM.pred_to_u8(q.numpy()), want)
    np.testing.assert_array_equal(IM.pred_to_u8(np.array([-3., -1e-7, 1. + 1e-7, 7.], np.float32)), [0, 0, 255, 255])


def test_gt_rule_recovers_stored_bytes():
    b = np.arange(256, dtype=np.uint8)
    np.testing.assert_array_equal(IM.gt_to_u8(b.astype(np.float32) / np.float32(255.)), b)
    np.testing.assert_array_equal(IM.gt_to_u8(np.array([-2., 0.4 / 255, 0.6 / 255, 1.2], np.float32)), [0, 0, 1, 255])


def test_host_side_of_image_metrics(golden):
    """eval.ssim_taps is rgb_ssim's filter, and eval.psnr_8bit is skimage's formula on the exact SSE, bit for bit."""
    from f2nerf_b200.eval import SSIM_TAPS, psnr_8bit
    assert SSIM_TAPS.dtype == np.float64 and SSIM_TAPS.shape == (11,)
    np.testing.assert_array_equal(SSIM_TAPS, IM.gaussian_taps())
    np.testing.assert_array_equal(SSIM_TAPS, SSIM_TAPS[::-1])
    for n in (str(n) for n in golden["names"]):
        gt, pred = golden[f"{n}_gt"], golden[f"{n}_pred"]
        assert psnr_8bit(IM.sse(pred, gt), gt.size) == float(golden[f"{n}_psnr"]), n
