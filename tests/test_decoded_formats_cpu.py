"""pigo_gray_images for *image.Gray16, RGBA64, NRGBA64, CMYK and Paletted without a device: the C and numpy restatements of
Go's colour models agree (exhaustively where the input space allows), they meet the conversions already pinned for the
8-bit formats, the arena size query counts the new formats, and every new invalid argument is refused before any device
work."""
import ctypes as C

import numpy as np
import pytest

import decoded_formats_oracle as F
import decoded_oracle as D
import oracle_lib as O
import pigo_b200
from pigo_b200 import DecodedImage, PIGO_E_CAP, PIGO_E_INVALID

GRAY16, RGBA64, NRGBA64, CMYK, PALETTED = 5, 6, 7, 8, 9


def _call(sources):
    descs = pigo_b200.decoded_descs(sources)
    imgs = (pigo_b200.PigoImage * max(len(sources), 1))()
    need = C.c_size_t(0)
    rc = pigo_b200.lib().pigo_gray_images(descs, len(sources), None, C.byref(need), imgs, pigo_b200.MEM_HOST, None)
    return rc, need.value


def _round256(x):
    return (x + 255) // 256 * 256


def _be16(v: np.ndarray) -> np.ndarray:
    """uint16 values [..., k] as the big-endian bytes [..., 2k] Go stores in Pix."""
    v = np.asarray(v, dtype=np.uint32)
    return np.stack([v >> 8, v & 0xFF], axis=-1).reshape(v.shape[:-1] + (2 * v.shape[-1],)).astype(np.uint8)


def _luma_both(nrgba_c, nrgba_np):
    g = O.rgba_to_gray(nrgba_c)
    assert np.array_equal(g, D.nrgba_luma_np(nrgba_np))
    return g


def test_constants_match_the_header():
    assert (pigo_b200.DECODED_GRAY16, pigo_b200.DECODED_RGBA64, pigo_b200.DECODED_NRGBA64, pigo_b200.DECODED_CMYK,
            pigo_b200.DECODED_PALETTED) == (GRAY16, RGBA64, NRGBA64, CMYK, PALETTED)


def test_gray16_restatements_agree_on_every_value_and_give_the_high_byte():
    y = np.arange(65536, dtype=np.uint32)[:, None]
    px = _be16(y)
    got_c, got_np = F.gray16_to_nrgba(px), F.gray16_to_nrgba_np(px)
    assert np.array_equal(got_c, got_np)
    hi = (y[:, 0] >> 8).astype(np.uint8)
    assert np.array_equal(_luma_both(got_c, got_np), hi)
    # y*0x101 is the Gray pixel y
    g = np.arange(256, dtype=np.uint8)
    rep = _be16(g.astype(np.uint32)[None, :] * 0x101)
    assert np.array_equal(F.decoded_gray(GRAY16, (rep.reshape(-1),), (512, 0), 256, 1), F.decoded_gray(3, (g,), (256, 0), 256, 1))


def test_cmyk_restatements_agree_on_every_channel_and_k_pair():
    c, k = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    px = np.stack([c, 255 - c, (c * 7) % 256, k], axis=-1).reshape(-1, 4).astype(np.uint8)
    got_c, got_np = F.cmyk_to_nrgba(px), F.cmyk_to_nrgba_np(px)
    assert np.array_equal(got_c, got_np)
    assert (got_c[:, 3] == 255).all()
    _luma_both(got_c, got_np)
    # K = 255 - g with no ink is the gray value g
    g = np.arange(256, dtype=np.uint8)
    ink = np.stack([np.zeros(256, np.uint8)] * 3 + [255 - g], axis=-1)
    assert np.array_equal(O.rgba_to_gray(F.cmyk_to_nrgba(ink)), g)


def _channel_cases(seed):
    """Every 16-bit alpha a crossed with the channels {0, 1, a-1, a, a+1, 0xffff} (clamped to 16 bits; each channel takes
    every value of the set once), plus a seeded sample of whole pixels."""
    a = np.arange(65536, dtype=np.int64)
    cand = [np.zeros_like(a), np.ones_like(a), np.maximum(a - 1, 0), a, np.minimum(a + 1, 0xFFFF), np.full_like(a, 0xFFFF)]
    rows = [np.stack([cand[j], cand[(j + 2) % 6], cand[(j + 4) % 6], a], axis=-1) for j in range(6)]
    rows.append(np.random.default_rng(seed).integers(0, 65536, size=(200000, 4)))
    return _be16(np.concatenate(rows).astype(np.uint32))


@pytest.mark.parametrize("premultiplied", [True, False], ids=["rgba64", "nrgba64"])
def test_rgba64_restatements_agree_on_every_alpha(premultiplied):
    px = _channel_cases(5 if premultiplied else 6)
    got_c, got_np = F.rgba64_to_nrgba(px, premultiplied), F.rgba64_to_nrgba_np(px, premultiplied)
    assert np.array_equal(got_c, got_np)
    _luma_both(got_c, got_np)
    a = px[:, 6].astype(int) * 256 + px[:, 7]
    assert not got_c[a == 0].any() and (got_c[a == 0xFFFF, 3] == 255).all()


def test_rgba64_with_replicated_bytes_is_the_rgba_path():
    c, a = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    px8 = np.stack([c, 255 - c, (c * 7) % 256, a], axis=-1).reshape(-1, 4).astype(np.uint8)
    px16 = _be16(px8.astype(np.uint32) * 0x101)
    want = D.rgba_to_nrgba(px8)
    assert np.array_equal(F.rgba64_to_nrgba(px16, True), want)
    assert np.array_equal(F.rgba64_to_nrgba_np(px16, True), want)


def test_opaque_nrgba64_gives_the_high_bytes():
    rgb = np.random.default_rng(8).integers(0, 65536, size=(4096, 3))
    v = np.concatenate([rgb, np.full((4096, 1), 0xFFFF)], axis=1).astype(np.uint32)
    got = F.rgba64_to_nrgba(_be16(v), False)
    assert np.array_equal(got[:, :3], (rgb >> 8).astype(np.uint8)) and (got[:, 3] == 255).all()
    assert np.array_equal(F.rgba64_to_nrgba_np(_be16(v), False), got)


def test_paletted_composition_and_indices_past_the_palette():
    pal = np.random.default_rng(9).integers(0, 256, size=(5, 4), dtype=np.uint8)
    idx = np.arange(12, dtype=np.uint8).reshape(3, 4)
    got = F.decoded_gray(PALETTED, (idx.reshape(-1), pal), (4, 5), 4, 3)
    want = O.rgba_to_gray(pal)[np.minimum(idx, 4)]
    want[idx >= 5] = 0
    assert np.array_equal(got, want)


def _sources():
    g16 = np.zeros((3, 9), np.uint8)        # 4 pixels of 2 bytes + 1 byte of padding
    p64 = np.zeros((2, 3, 8), np.uint8)
    cmyk = np.zeros((4, 5, 4), np.uint8)
    idx = np.zeros((6, 7), np.uint8)
    pal = np.zeros((3, 4), np.uint8)
    return [DecodedImage.gray16(g16, 4, 3), DecodedImage.rgba64(p64, 3, 2), DecodedImage.nrgba64(p64, 3, 1),
            DecodedImage.cmyk(cmyk, 5, 4), DecodedImage.paletted(idx, pal, 7, 6)]


def test_size_query_counts_the_new_formats_and_repeats_add_nothing():
    src = _sources()
    assert src[0].strides == (9, 0) and src[1].strides == (24, 0) and src[4].strides == (7, 3)
    want = _round256(12) + _round256(6) + _round256(3) + _round256(20) + _round256(42)
    assert _call(src) == (PIGO_E_CAP, want)
    assert pigo_b200.gray_images_bytes(src) == want
    assert _call(src + src[::-1] + [src[4]]) == (PIGO_E_CAP, want)
    # the palette pointer and length take part in the repeat test
    idx, pal = src[4].planes
    assert _call([src[4], DecodedImage.paletted(idx, pal[:2], 7, 6)])[1] == 2 * _round256(42)
    assert _call([src[4], DecodedImage.paletted(idx, pal.copy(), 7, 6)])[1] == 2 * _round256(42)


def _bad(which, **kw):
    s = _sources()[which]
    d = dict(format=s.format, width=s.width, height=s.height, planes=s.planes, strides=s.strides)
    d.update(kw)
    return DecodedImage(**d)


@pytest.mark.parametrize("which,bad", [
    (0, dict(format=10)), (0, dict(format=4)),
    (0, dict(strides=(7, 0))), (1, dict(strides=(23, 0))), (2, dict(strides=(23, 0))), (3, dict(strides=(19, 0))), (4, dict(strides=(6, 3))),
    (0, dict(planes=(None,))), (1, dict(planes=(None,))), (2, dict(planes=(None,))), (3, dict(planes=(None,))),
    (4, dict(planes=(None, np.zeros((3, 4), np.uint8)))),
    (4, dict(planes=(np.zeros(42, np.uint8), None))),
    (4, dict(strides=(7, 0))), (4, dict(strides=(7, 257))), (4, dict(strides=(7, -1))),
    (0, dict(width=0)), (4, dict(height=0)),
])
def test_new_invalid_arguments_fail_without_a_device(which, bad):
    assert _call(_sources() + [_bad(which, **bad)])[0] == PIGO_E_INVALID


def test_palette_lengths_one_and_256_are_accepted():
    idx = np.zeros((2, 2), np.uint8)
    for k in (1, 256):
        assert _call([DecodedImage.paletted(idx, np.zeros((k, 4), np.uint8), 2, 2)]) == (PIGO_E_CAP, 256)
