"""pigo_gray_images without a device: the arena size query, argument validation, and the oracle identities the GPU tests
rely on (the two RGBA -> NRGBA restatements agree; luma of an opaque gray pixel is the gray value)."""
import ctypes as C

import numpy as np
import pytest

import decoded_oracle as D
import oracle_lib as O
import pigo_b200
from oracle import np_oracle as N
from pigo_b200 import DecodedImage, PIGO_E_CAP, PIGO_E_INVALID, PIGO_OK


def _call(sources, gray=None, size=0, n=None):
    descs = pigo_b200.decoded_descs(sources)
    imgs = (pigo_b200.PigoImage * max(len(sources), 1))()
    need = C.c_size_t(size)
    rc = pigo_b200.lib().pigo_gray_images(descs, len(sources) if n is None else n, gray, C.byref(need), imgs, pigo_b200.MEM_HOST, None)
    return rc, need.value


def _round256(x):
    return (x + 255) // 256 * 256


def _sources():
    y = np.zeros((30, 41), np.uint8)
    cb = np.zeros((15, 21), np.uint8)
    rgba = np.zeros((7, 5, 4), np.uint8)
    g = np.zeros((1, 1), np.uint8)
    return [DecodedImage.ycbcr(y, cb, cb, 2, 40, 29, min_x=1, min_y=1), DecodedImage.nrgba(rgba, 5, 7), DecodedImage.rgba(rgba, 5, 6),
            DecodedImage.gray(g, 1, 1)]


def test_size_query_needs_no_device_and_repeats_add_nothing():
    src = _sources()
    want = _round256(40 * 29) + _round256(35) + _round256(30) + _round256(1)
    assert _call(src) == (PIGO_E_CAP, want)
    assert pigo_b200.gray_images_bytes(src) == want
    assert _call(src + src[::-1] + [src[2]]) == (PIGO_E_CAP, want)       # byte-identical descriptors share a slot
    assert _call(src, gray=1 << 40, size=want - 1) == (PIGO_E_CAP, want)  # too small: reported before any device call
    assert _call([]) == (PIGO_OK, 0)
    # a different stride or origin is a different source
    y = src[0].planes[0]
    other = DecodedImage.ycbcr(y, src[0].planes[1], src[0].planes[2], 2, 40, 29, min_x=1, min_y=1, y_stride=40)
    assert _call([src[0], other])[1] == 2 * _round256(40 * 29)
    assert _call([src[0], DecodedImage.ycbcr(y, src[0].planes[1], src[0].planes[2], 2, 40, 29, min_x=2, min_y=1)])[1] == 2 * _round256(40 * 29)


def _bad(**kw):
    s = _sources()[kw.pop("which", 0)]
    d = dict(format=s.format, width=s.width, height=s.height, planes=s.planes, strides=s.strides, subsample=s.subsample, min_x=s.min_x, min_y=s.min_y)
    d.update(kw)
    return DecodedImage(**d)


@pytest.mark.parametrize("bad", [
    dict(format=4), dict(format=-1),
    dict(subsample=6), dict(subsample=-1),
    dict(min_x=-1), dict(min_y=-2),
    dict(width=0), dict(height=0), dict(which=1, width=-3),
    dict(which=3, width=65536, height=32768, strides=(65536, 0)),
    dict(strides=(39, 21)), dict(strides=(40, 19)), dict(which=1, strides=(19, 0)), dict(which=2, strides=(19, 0)), dict(which=3, strides=(0, 0)),
    dict(planes=(None, np.zeros(8, np.uint8), np.zeros(8, np.uint8))), dict(planes=(np.zeros(8, np.uint8), None, np.zeros(8, np.uint8))),
    dict(planes=(np.zeros(8, np.uint8), np.zeros(8, np.uint8), None)), dict(which=1, planes=(None,)), dict(which=3, planes=(None,)),
])
def test_invalid_arguments_fail_without_a_device(bad):
    assert _call(_sources() + [_bad(**bad)])[0] == PIGO_E_INVALID


def test_invalid_counts_and_pointers():
    src = _sources()
    assert _call(src, n=-1)[0] == PIGO_E_INVALID
    assert _call(src * 16384 + src[:1], n=65536)[0] == PIGO_E_INVALID
    assert _call(src * 16384, n=65535)[0] == PIGO_E_CAP                       # 65535 sources are allowed
    L = pigo_b200.lib()
    need = C.c_size_t(0)
    assert L.pigo_gray_images(None, 1, None, C.byref(need), (pigo_b200.PigoImage * 1)(), 0, None) == PIGO_E_INVALID
    assert L.pigo_gray_images(pigo_b200.decoded_descs(src), 1, None, C.byref(need), None, 0, None) == PIGO_E_INVALID
    assert L.pigo_gray_images(pigo_b200.decoded_descs(src), 1, None, None, (pigo_b200.PigoImage * 1)(), 0, None) == PIGO_E_INVALID


def test_nrgba_model_restatements_agree_on_every_channel_alpha_pair():
    c, a = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    px = np.stack([c, 255 - c, (c * 7) % 256, a], axis=-1).reshape(-1, 4).astype(np.uint8)
    got_c, got_np = D.rgba_to_nrgba(px), D.rgba_to_nrgba_np(px)
    assert np.array_equal(got_c, got_np)
    opaque, clear = px[:, 3] == 255, px[:, 3] == 0
    assert np.array_equal(got_c[opaque], px[opaque]) and not got_c[clear].any()
    # valid premultiplied input (channel <= alpha) comes back within one step of the straight value
    ok = (px[:, 0].astype(int) <= px[:, 3]) & ~clear
    straight = px[ok, 0].astype(int) * 255 / px[ok, 3]
    assert np.all(np.abs(got_c[ok, 0] - straight) <= 1.0)
    # the luma of the converted pixels is the same through either gray restatement
    assert np.array_equal(O.rgba_to_gray(got_c), D.nrgba_luma_np(got_np))


def test_luma_of_an_opaque_gray_pixel_is_its_value():
    y = np.arange(256, dtype=np.uint8)
    px = np.stack([y, y, y, np.full(256, 255, np.uint8)], axis=-1)
    assert np.array_equal(O.rgba_to_gray(px), y)
    assert np.array_equal(D.nrgba_luma_np(px), y)
    assert np.array_equal(N.rgb_to_grayscale(px[:, :3]), y)


def test_oracle_composition_of_each_format():
    rng = np.random.default_rng(3)
    px = rng.integers(0, 256, size=(5, 6, 4), dtype=np.uint8)
    flat = np.concatenate([px.reshape(5, 24), np.zeros((5, 4), np.uint8)], axis=1).reshape(-1)   # Stride 28 > 24
    assert np.array_equal(D.decoded_gray(1, (flat,), (28, 0), 6, 5), O.rgba_to_gray(px))
    assert np.array_equal(D.decoded_gray(2, (flat,), (28, 0), 6, 5), O.rgba_to_gray(D.rgba_to_nrgba_np(px)))
    g = rng.integers(0, 256, size=(4, 9), dtype=np.uint8)
    assert np.array_equal(D.decoded_gray(3, (g.reshape(-1),), (9, 0), 7, 4), g[:, :7])
    y, cb, cr = O.make_ycbcr_planes(4, 2, 11, 7, 1, 3)
    want = O.rgba_to_gray(O.ycbcr_to_nrgba(y, cb, cr, 2, 11, 7, 1, 3))
    assert np.array_equal(D.decoded_gray(0, (y, cb, cr), (y.shape[1], cb.shape[1]), 11, 7, 2, 1, 3), want)
