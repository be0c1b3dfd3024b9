"""Splatter(..., primitive) argument checks (CPU: refused before any device work)."""
import pytest

from helpers import scene


def _make(**kw):
    import splatter
    g, v, _ = scene(50, 32, 32, sh_dim=kw.pop("sh_dim", 3))
    vs = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)]
    return splatter.Splatter.from_tensors(g, vs, device="cpu", **kw)


@pytest.mark.parametrize("bad", ["disk", "Surfel", None, 2])
def test_primitive_must_be_gaussian_or_surfel(bad):
    with pytest.raises(ValueError, match="primitive"):
        _make(primitive=bad)


@pytest.mark.parametrize("kw", [dict(filter2d="antialias"), dict(filter3d=True), dict(densify_stats="grad"),
                                dict(n_features=8), dict(camera_model="colmap")])
def test_surfels_refuse_what_they_have_no_kernel_for(kw):
    with pytest.raises(ValueError, match="primitive='surfel' does not take " + next(iter(kw))):
        _make(primitive="surfel", **kw)


def test_surfels_refuse_per_pixel_sh():
    with pytest.raises(ValueError, match="sh_eval='gaussian'"):
        _make(primitive="surfel", sh_dim=27, use_sh_coeff=True)
