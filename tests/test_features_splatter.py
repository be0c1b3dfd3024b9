"""Splatter(..., n_features) argument checks (CPU: refused before any device work)."""
import pytest
import torch

from helpers import scene


def _make(**kw):
    import splatter
    g, v, _ = scene(50, 32, 32, sh_dim=kw.pop("sh_dim", 3))
    if "feat" in kw:
        g["feat"] = kw.pop("feat")
    vs = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)]
    return splatter.Splatter.from_tensors(g, vs, device="cpu", **kw)


@pytest.mark.parametrize("bad", [4, 12, 64, -8, "16"])
def test_n_features_must_be_8_16_or_32(bad):
    with pytest.raises(ValueError, match="n_features"):
        _make(n_features=bad)


def test_features_refused_with_per_pixel_sh():
    with pytest.raises(ValueError, match="per-pixel SH"):
        _make(n_features=16, sh_dim=27, use_sh_coeff=True)


def test_features_refused_with_absgrad():
    with pytest.raises(ValueError, match="absgrad"):
        _make(n_features=8, densify_stats="absgrad")


def test_feature_tensor_width_sets_and_must_match_n_features():
    with pytest.raises(ValueError, match="n_features"):
        _make(feat=torch.zeros(50, 12))                     # inferred width 12 is not a supported width
    with pytest.raises(ValueError, match=r"\[n, n_features\]"):
        _make(feat=torch.zeros(50, 8), n_features=16)
