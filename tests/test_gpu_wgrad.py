"""The weight gradient (vp_conv_wgrad) on one-hot operands: a single nonzero x element and a single nonzero dy element that
some filter tap pairs must give exactly one nonzero dW element, at that (tap, dy channel, x channel), with the exact product
as its value; every other element of the packed buffer, padding included, stays exactly as it was.  This pins down the
kernel's index bookkeeping on its own: which channel each GEMM row holds, which tap each row block belongs to, the
stride-parity maps of the shifted operand, the tile order of the transposed copy of the other operand, the transposed
store of a conv's dW and the pixel-range splits.  The channels of
both operands outside their views hold NaN and must not be read."""
import random
import zlib

import pytest
import torch

gpu = pytest.mark.gpu
NAN = float('nan')

# (k, s, p, transposed, ci, co, input extent (d, h, w), batch): every stride pattern of the model (1, (1,2,2), (2,2,2),
# transposed (1,2,2)), odd extents that give parity lattices of unequal size, partial tiles, and channel counts that use
# several 32-channel dy chunks, several x-channel tiles and each N tile width
CASES = [
    ((1, 5, 5), (1, 1, 1), (0, 2, 2), False, 72, 128, (1, 32, 32), 3),
    ((1, 5, 5), (1, 1, 1), (0, 2, 2), False, 264, 512, (1, 8, 8), 2),
    ((1, 5, 5), (1, 1, 1), (0, 2, 2), False, 136, 256, (1, 6, 6), 3),
    ((1, 3, 3), (1, 1, 1), (0, 1, 1), False, 60, 7, (1, 9, 7), 5),
    ((1, 3, 3), (1, 1, 1), (0, 1, 1), False, 32, 3, (1, 12, 10), 2),
    ((1, 4, 4), (1, 2, 2), (0, 1, 1), False, 40, 80, (1, 13, 11), 3),
    ((1, 6, 6), (1, 2, 2), (0, 2, 2), False, 16, 32, (1, 16, 16), 2),
    ((4, 4, 4), (1, 2, 2), (1, 1, 1), False, 32, 64, (5, 16, 16), 2),
    ((4, 4, 4), (2, 2, 2), (1, 1, 1), False, 24, 48, (9, 13, 11), 2),
    ((3, 3, 3), (1, 1, 1), (1, 1, 1), False, 128, 128, (4, 8, 8), 2),
    ((1, 6, 6), (1, 2, 2), (0, 2, 2), True, 136, 64, (1, 8, 8), 3),
    ((1, 6, 6), (1, 2, 2), (0, 2, 2), True, 40, 48, (1, 5, 7), 2),
]


def out_extent(k, s, p, transposed, ext):
    if transposed:
        return tuple((i - 1) * ss - 2 * pp + kk for i, ss, pp, kk in zip(ext, s, p, k))
    return tuple((i + 2 * pp - kk) // ss + 1 for i, ss, pp, kk in zip(ext, s, p, k))


def case_id(c):
    k, s, p, t, ci, co, ext, n = c
    return 'k%s_s%s_%sci%d_co%d_%s_n%d' % (''.join(map(str, k)), ''.join(map(str, s)), 'T' if t else '', ci, co,
                                           'x'.join(map(str, ext)), n)


@pytest.fixture(scope='module')
def L():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from video_prediction_b200 import lib
    lib.lib()
    return lib


def pairs(case, rng, count):
    """`count` random (x pixel, dy pixel, tap) triples that the geometry connects: conv reads x at s*o + r - p for output o,
    a transposed conv writes dy at s*i + r - p for input i."""
    k, s, p, transposed, ci, co, ext, n = case
    oext = out_extent(k, s, p, transposed, ext)
    out = []
    while len(out) < count:
        b = rng.randrange(n)
        r = tuple(rng.randrange(kk) for kk in k)
        if transposed:
            i = tuple(rng.randrange(e) for e in ext)
            o = tuple(ss * ii + rr - pp for ss, ii, rr, pp in zip(s, i, r, p))
        else:
            o = tuple(rng.randrange(e) for e in oext)
            i = tuple(ss * oo + rr - pp for ss, oo, rr, pp in zip(s, o, r, p))
        if all(0 <= v < e for v, e in zip(i, ext)) and all(0 <= v < e for v, e in zip(o, oext)):
            out.append(((b,) + i, (b,) + o, (r[0] * k[1] + r[1]) * k[2] + r[2]))
    return out


@gpu
@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_wgrad_one_hot(L, case):
    k, s, p, transposed, ci, co, ext, n = case
    oext = out_extent(k, s, p, transposed, ext)
    taps = k[0] * k[1] * k[2]
    wp_n_pad = L.choose_n_pad(co)
    kc = (ci + 31) // 32
    g = L.geom(k, s, p, transposed)
    rng = random.Random(zlib.crc32(case_id(case).encode()))
    x = torch.full((n,) + tuple(ext) + (ci + 4,), NAN, device='cuda')
    dy = torch.full((n,) + tuple(oext) + ((co + 3) // 4 * 4 + 4,), NAN, device='cuda')
    # small integers: adding the product to them and subtracting them again is exact
    base = torch.randint(-8, 8, (taps * wp_n_pad * kc * 32,), generator=torch.Generator().manual_seed(0)).float().cuda()
    for xi, oi, tap in pairs(case, rng, 6):
        cx, cy = rng.randrange(ci), rng.randrange(co)
        x[..., :ci] = 0.0
        dy[..., :co] = 0.0
        x[xi + (cx,)] = 1.5
        dy[oi + (cy,)] = -2.25
        for split in (0, 1, 3):
            dwp = base.clone()
            L.conv_wgrad(L.tensor_view(x, ci), L.tensor_view(dy, co), g, dwp, wp_n_pad, kc, split)
            diff = (dwp - base).view(taps, wp_n_pad, kc * 32)
            nz = diff.nonzero().tolist()
            where = 'x %s c%d, dy %s c%d, tap %d, split %d' % (xi, cx, oi, cy, tap, split)
            assert nz == [[tap, cy, cx]], where + ': nonzero at %s' % nz[:8]
            assert diff[tap, cy, cx].item() == 1.5 * -2.25, where
