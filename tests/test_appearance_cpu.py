"""Appearance arguments without a GPU (DESIGN.md §3m): ``Renderer.appearance_row`` resolves None / an index / a [16] row / "own"
and refuses everything else; ``TestAppearance``'s half-image split; ``RenderPath``'s per-frame rows."""
import numpy as np
import pytest
import torch


def renderer(use_app_emb=True, n_images=5):
    from f2nerf_b200 import GlobalDataPool, Hash3DAnchored, Renderer, SHShader
    gdp = GlobalDataPool()
    return Renderer(gdp, None, Hash3DAnchored(gdp, log2_table_size=8, device="cpu"), SHShader(gdp, device="cpu"), n_images=n_images,
                    use_app_emb=use_app_emb, device="cpu")


def test_appearance_row_resolution():
    r = renderer()
    assert r.appearance_row(None) is None
    for i in (0, 4, np.int64(2)):
        row = r.appearance_row(i)
        assert row.shape == (16,) and row.dtype == torch.float32 and torch.equal(row, r.app_emb_.detach()[int(i)])
        assert row.data_ptr() != r.app_emb_.data_ptr()                       # a copy: later writes to app_emb_ do not reach it
    assert torch.equal(r.appearance_row("own", view=3), r.app_emb_.detach()[3])
    assert r.appearance_row(None, view=3) is None
    given = torch.arange(16, dtype=torch.float64) / 7.
    row = r.appearance_row(given)
    assert row.dtype == torch.float32 and row.is_contiguous() and torch.equal(row, given.float())
    assert torch.equal(r.appearance_row(given.tolist()), given.float())
    strided = torch.arange(32, dtype=torch.float32)[::2]
    assert r.appearance_row(strided).is_contiguous() and torch.equal(r.appearance_row(strided), strided)


@pytest.mark.parametrize("bad, match", [(5, "outside"), (-1, "outside"), (np.int32(9), "outside"), (True, "bool"),
                                        (torch.zeros(15), "16 entries"), (torch.zeros(1, 16), "16 entries"), (torch.zeros(()), "16 entries"),
                                        (0.5, "16 entries"), ("mine", "unknown"), ("own", "needs a view")])
def test_appearance_row_refusals(bad, match):
    with pytest.raises(ValueError, match=match):
        renderer().appearance_row(bad)


def test_renderer_without_embedding_refuses_every_appearance():
    r = renderer(use_app_emb=False)
    assert r.appearance_row(None) is None and r.appearance_row(None, view=1) is None
    for a in (0, torch.zeros(16), "own"):
        with pytest.raises(ValueError, match="use_app_emb"):
            r.appearance_row(a, view=1)


def test_half_image_split():
    from f2nerf_b200.appearance import left_half_mask, right_half_pixels
    for H, W in ((4, 7), (5, 8), (3, 1), (540, 960)):
        left = left_half_mask(H, W)
        right = right_half_pixels(H, W)
        assert left.shape == (H, W) and left.dtype == torch.bool
        assert bool(left[:, :W // 2].all()) and not bool(left[:, W // 2:].any())
        flat = torch.zeros(H * W, dtype=torch.int32)
        flat[right] += 1
        flat[torch.nonzero(left.reshape(-1)).squeeze(1)] += 1
        assert bool((flat == 1).all())                                      # the two halves partition the image
        img = torch.arange(H * W * 3).reshape(H, W, 3)
        assert torch.equal(img.reshape(-1, 3)[right].reshape(H, W - W // 2, 3), img[:, W // 2:])   # row-major order of the crop


def test_path_rows():
    from f2nerf_b200.eval import path_rows
    r = renderer()
    assert path_rows(r, None, 3) == [None, None, None]
    rows = path_rows(r, 2, 3)
    assert len(rows) == 3 and all(torch.equal(x, r.app_emb_.detach()[2]) for x in rows)
    a, b = r.app_emb_.detach()[0], r.app_emb_.detach()[1]
    s = torch.linspace(0., 1., 4)[:, None]
    blend = (1. - s) * a + s * b                                           # the caller's blend of two looks, one row per frame
    rows = path_rows(r, blend, 4)
    assert len(rows) == 4 and all(torch.equal(x, blend[f]) for f, x in enumerate(rows))
    for bad in (torch.zeros(3, 16), torch.zeros(4, 15), torch.zeros(5, 16)):
        with pytest.raises(ValueError, match="per-frame"):
            path_rows(r, bad, 4)
    with pytest.raises(ValueError, match="needs a view"):
        path_rows(r, "own", 4)
    with pytest.raises(ValueError, match="use_app_emb"):
        path_rows(renderer(use_app_emb=False), blend, 4)
