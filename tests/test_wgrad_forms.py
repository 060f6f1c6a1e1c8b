"""The weight gradient's launch plan (lib.conv_wgrad_form) for every distinct wgrad call of the cfg2 training step (SAVP,
B = 16, 2 + 10 frames) on a 132-SM H100, without a device.  The pixel-range split count groups every dW sum, so it must
stay that of the layer's rule (two waves of taps x 128-row dy tiles x 128-column x tiles, at least four 64-pixel tiles per
split) whatever form the call runs in; the form's CTA count must be its (row-block groups x column tiles x splits)."""
import pytest

from video_prediction_b200 import lib as L

SMS = 132

# (x (n, d, h, w, c), dy (n, d, h, w, c), geometry (k, s, p, transposed), n_pad, kc) of the cfg2 step's wgrad calls
CALLS = [
    ((176, 1, 16, 16, 128), (176, 1, 8, 8, 256), (1, 4, 4, 1, 2, 2, 0, 1, 1, 0), 256, 4),
    ((176, 1, 32, 32, 64), (176, 1, 16, 16, 128), (1, 4, 4, 1, 2, 2, 0, 1, 1, 0), 128, 2),
    ((176, 1, 64, 64, 8), (176, 1, 32, 32, 64), (1, 4, 4, 1, 2, 2, 0, 1, 1, 0), 64, 1),
    ((32, 10, 64, 64, 32), (32, 9, 32, 32, 64), (4, 4, 4, 1, 2, 2, 1, 1, 1, 0), 64, 1),
    ((32, 4, 8, 8, 256), (32, 4, 8, 8, 256), (3, 3, 3, 1, 1, 1, 1, 1, 1, 0), 256, 8),
    ((32, 8, 16, 16, 128), (32, 4, 8, 8, 256), (4, 4, 4, 2, 2, 2, 1, 1, 1, 0), 256, 4),
    ((32, 8, 16, 16, 128), (32, 8, 16, 16, 128), (3, 3, 3, 1, 1, 1, 1, 1, 1, 0), 128, 4),
    ((32, 9, 32, 32, 64), (32, 8, 16, 16, 128), (4, 4, 4, 1, 2, 2, 1, 1, 1, 0), 128, 2),
    ((32, 9, 32, 32, 64), (32, 9, 32, 32, 64), (3, 3, 3, 1, 1, 1, 1, 1, 1, 0), 64, 2),
    ((352, 1, 16, 16, 136), (352, 1, 16, 16, 256), (1, 5, 5, 1, 1, 1, 0, 2, 2, 0), 256, 5),
    ((352, 1, 16, 16, 136), (352, 1, 32, 32, 32), (1, 6, 6, 1, 2, 2, 0, 2, 2, 1), 32, 5),
    ((352, 1, 16, 16, 72), (352, 1, 8, 8, 128), (1, 4, 4, 1, 2, 2, 0, 1, 1, 0), 128, 3),
    ((352, 1, 32, 32, 40), (352, 1, 16, 16, 64), (1, 4, 4, 1, 2, 2, 0, 1, 1, 0), 64, 2),
    ((352, 1, 32, 32, 72), (352, 1, 32, 32, 128), (1, 5, 5, 1, 1, 1, 0, 2, 2, 0), 128, 3),
    ((352, 1, 32, 32, 72), (352, 1, 64, 64, 32), (1, 6, 6, 1, 2, 2, 0, 2, 2, 1), 32, 3),
    ((352, 1, 64, 64, 16), (352, 1, 32, 32, 32), (1, 6, 6, 1, 2, 2, 0, 2, 2, 0), 32, 1),
    ((352, 1, 64, 64, 32), (352, 1, 64, 64, 3), (1, 3, 3, 1, 1, 1, 0, 1, 1, 0), 16, 1),
    ((352, 1, 64, 64, 32), (352, 1, 64, 64, 32), (1, 3, 3, 1, 1, 1, 0, 1, 1, 0), 32, 1),
    ((352, 1, 64, 64, 60), (352, 1, 64, 64, 7), (1, 3, 3, 1, 1, 1, 0, 1, 1, 0), 16, 2),
    ((352, 1, 8, 8, 136), (352, 1, 16, 16, 64), (1, 6, 6, 1, 2, 2, 0, 2, 2, 1), 64, 5),
    ((352, 1, 8, 8, 264), (352, 1, 8, 8, 512), (1, 5, 5, 1, 1, 1, 0, 2, 2, 0), 512, 9),
]


def cdiv(a, b):
    return -(-a // b)


def floor_pow2(v):
    p = 1
    while p * 2 <= v:
        p *= 2
    return p


def rule(x, dy, geo, n_pad, kc, sms):
    """(64-pixel tiles, split count) of the layer's rule, split_k = 0."""
    plain = x if geo[9] else dy
    rem, tiles = 64, 1
    for e in (plain[3], plain[2], plain[1]):         # w, h, d: powers of two, w fastest
        b = min(floor_pow2(e), rem)
        rem //= b
        tiles *= cdiv(e, b)
    tiles *= cdiv(plain[0], rem)
    taps = geo[0] * geo[1] * geo[2]
    ctas = taps * cdiv(min(n_pad, cdiv(dy[4], 32) * 32), 128) * cdiv(kc, 4)
    return tiles, max(1, min(max(1, 2 * sms // ctas), max(1, tiles // 4)))


@pytest.mark.parametrize('call', CALLS, ids=['x%s_dy%s' % ('x'.join(map(str, c[0])), 'x'.join(map(str, c[1]))) for c in CALLS])
def test_split_count_is_the_layers_and_ctas_are_reported(call):
    x, dy, geo, n_pad, kc = call
    form, ctas, splits, stages = L.conv_wgrad_form(L.VpConvGeom(*geo), x, dy, n_pad, kc, SMS, 0)
    tiles, want = rule(x, dy, geo, n_pad, kc, SMS)
    assert splits == want
    assert stages == cdiv(tiles, splits)
    blocks, bn = L.conv_wgrad_forms()[form]
    shifted_c, plain_c = (dy[4], x[4]) if geo[9] else (x[4], dy[4])
    assert ctas == cdiv(geo[0] * geo[1] * geo[2] * cdiv(shifted_c, 32), blocks) * cdiv(plain_c, bn) * splits
    print('%s: %d blocks x %d columns, %d CTAs (%.2f waves), %d splits, %d stages per CTA'
          % (call, blocks, bn, ctas, ctas / SMS, splits, stages))
