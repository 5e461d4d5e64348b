"""Argument checks of coarse embedding images (RGBDImages(..., upsample_embeddings=True)), raised on the host before any
CUDA call: the keyword's refusals, the coarse shapes it accepts, the flag through the container operations, and the
refusals of the three upsampled C entry points."""
import pytest
import torch

import gradslam_b200 as gs
from gradslam_b200 import _C


def _frames(B=2, L=1, H=4, W=5, emb=None, channels_first=False, **kw):
    if channels_first:
        rgb, depth = torch.rand(B, L, 3, H, W), torch.rand(B, L, 1, H, W)
    else:
        rgb, depth = torch.rand(B, L, H, W, 3), torch.rand(B, L, H, W, 1)
    K = torch.eye(4).repeat(B, 1, 1, 1)
    poses = torch.eye(4).repeat(B, L, 1, 1)
    return gs.RGBDImages(rgb, depth, K, poses, channels_first=channels_first, embeddings=emb, **kw)


@pytest.mark.parametrize("shape", [(2, 1, 1, 1, 3), (2, 1, 2, 3, 7), (2, 1, 4, 5, 1), (2, 1, 1, 5, 2), (2, 1, 4, 1, 2)])
def test_keyword_accepts_coarse_images(shape):
    e = torch.rand(shape)
    f = _frames(emb=e, upsample_embeddings=True)
    assert f.upsample_embeddings is True and f.embeddings is e
    cf = torch.rand(2, 1, shape[4], shape[2], shape[3], dtype=torch.float16)
    g = _frames(emb=cf, channels_first=True, upsample_embeddings=True)
    assert g.upsample_embeddings and g.embeddings.shape == cf.shape


def test_default_is_off_and_full_resolution_images_are_checked_as_before():
    f = _frames(emb=torch.rand(2, 1, 4, 5, 3))
    assert f.upsample_embeddings is False
    assert _frames().upsample_embeddings is False
    with pytest.raises(ValueError):  # a coarse image needs the keyword
        _frames(emb=torch.rand(2, 1, 2, 3, 3))


@pytest.mark.parametrize("kw, err", [
    (dict(upsample_embeddings=True), ValueError),  # no embeddings
    (dict(emb=torch.rand(2, 1, 2, 3, 3), upsample_embeddings=1), TypeError),
    (dict(emb=torch.rand(2, 1, 2, 3, 3), upsample_embeddings=None), TypeError),
    (dict(emb=torch.rand(2, 1, 5, 3, 3), upsample_embeddings=True), ValueError),  # h > H
    (dict(emb=torch.rand(2, 1, 2, 6, 3), upsample_embeddings=True), ValueError),  # w > W
    (dict(emb=torch.rand(2, 1, 0, 3, 3), upsample_embeddings=True), ValueError),  # h = 0
    (dict(emb=torch.rand(2, 1, 2, 0, 3), upsample_embeddings=True), ValueError),  # w = 0
    (dict(emb=torch.rand(2, 1, 2, 3, 0), upsample_embeddings=True), ValueError),  # D = 0
    (dict(emb=torch.rand(1, 1, 2, 3, 3), upsample_embeddings=True), ValueError),  # B
    (dict(emb=torch.rand(2, 2, 2, 3, 3), upsample_embeddings=True), ValueError),  # L
    (dict(emb=torch.rand(2, 1, 2, 3), upsample_embeddings=True), ValueError),  # ndim
    (dict(emb=torch.rand(2, 1, 2, 3, 3).double(), upsample_embeddings=True), TypeError),
    (dict(emb=[[0.0]], upsample_embeddings=True), TypeError),
])
def test_keyword_refusals(kw, err):
    emb = kw.pop("emb", None)
    with pytest.raises(err):
        _frames(emb=emb, **kw)


def test_channels_first_frames_refuse_a_channels_last_coarse_image():
    with pytest.raises(ValueError):  # (2, 1, 2, 3, 7): D = 2 would be read as channels, (h, w) = (3, 7) > (4, 5)
        _frames(emb=torch.rand(2, 1, 2, 3, 7), channels_first=True, upsample_embeddings=True)


def test_flag_survives_the_container_operations():
    e = torch.rand(2, 3, 2, 3, 7)
    f = _frames(L=3, emb=e, upsample_embeddings=True)
    for g in (f[:, 1], f[1], f[0, 0:2], f.clone(), f.detach(), f.to("cpu", copy=True)):
        assert g.upsample_embeddings is True
        assert tuple(g.embeddings.shape[2:]) == (2, 3, 7)
    cf = f.to_channels_first()
    assert cf.upsample_embeddings and cf.embeddings.shape == (2, 3, 7, 2, 3)
    back = cf.to_channels_last()
    assert back.upsample_embeddings and torch.equal(back.embeddings, e)
    kept = gs.RGBDImages(f.rgb_image, f.depth_image, f.intrinsics, f.poses, embeddings=f.embeddings,
                         upsample_embeddings=f.upsample_embeddings)  # the constructor bilateral_filtered uses
    assert kept.upsample_embeddings and kept.embeddings is e
    plain = _frames(L=3, emb=torch.rand(2, 3, 4, 5, 7))
    assert not plain[:, 1].upsample_embeddings and not plain.clone().upsample_embeddings


def test_bilateral_filtered_passes_the_flag(monkeypatch):
    from gradslam_b200.structures import rgbdimages as rgbd

    monkeypatch.setattr(rgbd, "bilateral_filter_depth", lambda d, f: d.clone())  # (the filter itself needs CUDA)
    f = _frames(emb=torch.rand(2, 1, 2, 3, 4), upsample_embeddings=True)
    g = f.bilateral_filtered(gs.BilateralFilter(2, 3.0, 0.05))
    assert g.upsample_embeddings and g.embeddings is f.embeddings


# ---- the C entry points (no launch happens: every call below is refused before one)
def _err():
    return _C.lib().gsx_last_error().decode()


_PTR = 1 << 20  # a 16-byte aligned stand-in address; never dereferenced by a refused call


def _fwd(eh=2, ew=3, stride=None, ptrs=(_PTR,) * 4, B=1, H=4, W=5, D=8, dtype=0):
    stride = eh * ew * D if stride is None else stride
    return _C.lib().gsx_embed_merge_append_upsampled(ptrs[0], 100, ptrs[1], stride, ptrs[2], ptrs[3], B, H, W, eh, ew,
                                                     D, dtype, None)


def _bwd(eh=2, ew=3, ptrs=(_PTR,) * 9, B=1, H=4, W=5, D=8):
    p = ptrs
    return _C.lib().gsx_embed_merge_bwd_upsampled(p[0], p[1], p[2], p[3], 10, p[4], p[5], 20, B, H, W, eh, ew, D, p[6],
                                                  p[7], p[8], p[8], None)


def _seq(eh=2, ew=3, ptrs=(_PTR,) * 4, D=8, dtype=0):
    p = ptrs
    return _C.lib().gsx_pointfusion_sequence_gt_emb_upsampled(
        _PTR, _PTR, _PTR, 100, 0, _PTR, _PTR, _PTR, _PTR, 1, 2, 0, 2, 4, 5, 0.05, 0.9, 0.6, _PTR, _PTR, 0, p[0], p[1],
        eh, ew, D, dtype, p[2], p[3], None)


@pytest.mark.parametrize("eh, ew", [(0, 3), (5, 3), (2, 0), (2, 6), (-1, 1)])
def test_c_entry_points_refuse_an_image_outside_the_depth(eh, ew):
    for call in (_fwd, _bwd, _seq):
        assert call(eh=eh, ew=ew) == 1
        assert "embedding image" in _err()


def test_c_entry_points_refuse_a_short_stride():
    assert _fwd(stride=2 * 3 * 8 - 1) == 1
    assert "stride" in _err()


@pytest.mark.parametrize("i", range(4))
def test_c_entry_points_refuse_null_pointers(i):
    ptrs = [_PTR] * 4
    ptrs[i] = None
    assert _fwd(ptrs=ptrs) == 1 and "null" in _err()
    assert _seq(ptrs=ptrs) == 1 and "null" in _err()
    bptrs = [_PTR] * 9
    bptrs[[0, 1, 4, 7][i]] = None
    assert _bwd(ptrs=bptrs) == 1 and "null" in _err()


def test_c_entry_points_refuse_misaligned_pointers():
    for i in range(4):
        ptrs = [_PTR] * 4
        ptrs[i] = _PTR + 1
        assert _fwd(ptrs=ptrs, dtype=1) == 1 and "misaligned" in _err()
    assert _fwd(ptrs=(_PTR, _PTR + 2, _PTR, _PTR), dtype=0) == 1 and "misaligned" in _err()
    assert _seq(ptrs=(_PTR + 1, _PTR, _PTR, _PTR), dtype=1) == 1 and "misaligned" in _err()
    assert _seq(ptrs=(_PTR, _PTR, _PTR, _PTR + 4), dtype=0) == 1 and "misaligned" in _err()
    assert _seq(ptrs=(_PTR, _PTR, _PTR + 2, _PTR), dtype=0) == 1 and "misaligned" in _err()
    for i in range(9):
        bptrs = [_PTR] * 9
        bptrs[i] = _PTR + (4 if i == 1 else 2)  # (merge_rec needs 8 bytes, the rest 4)
        assert _bwd(ptrs=bptrs) == 1 and "misaligned" in _err()
