"""The forward / dgrad kernel of the engine (igemm_fwd_kernel) at batches where a CTA walks several pixel tiles.

A CTA of that kernel is persistent over the 128-pixel tiles blockIdx.x, blockIdx.x + gridDim.x, ...; one ring of
shared-memory stages streams across its tiles, and its consumers release each stage while the next chunk's MMAs are in
flight.  tests/test_gpu_engine.py runs every model geometry at batch 1-2, where almost every CTA holds a single tile, so
the ring positions and phases of a CTA's later tiles are exercised here: at batches that give 1, 2, 3 and 5 tiles per CTA,
every call is checked against the fp64 reference of tests/test_gpu_engine.py, and the full batch must equal, bit for bit,
the same call run on batch slices small enough that every CTA holds a single tile: a tile's result must not depend on
which CTA computed it or where in the ring its stages were."""
import pytest
import torch

import test_gpu_engine as E
from test_gpu_conv_lstm import _cell64, _lstm_case
from test_gpu_engine import L, mode  # noqa: F401  (fixtures of the engine check)
from test_gpu_engine import PLAIN, S1, S2, UPSAMPLED, _case

pytestmark = pytest.mark.gpu
NAN = float('nan')
TILES_PER_CTA = (1, 2, 3, 5)

CASES = [
    # BN 32, kc 1: 9 k-chunks per tile against a ring of 8 stages
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 32, 32, (1, 16, 16)),
    # BN 64, k_tail 1 (40 channels = 32 + 8)
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 40, 48, (1, 8, 8)),
    # BN 128
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 64, 128, (1, 8, 8)),
    # transposed: four output phases (the generator's upsample_conv2d)
    _case(UPSAMPLED, (1, 3, 3), S2, (0, 2, 2), True, 72, 32, (1, 8, 8)),
]


def _pow2_floor(v):
    return 1 << (max(v, 1).bit_length() - 1)


def launch(lat, n, n_pad, phases, bn=None):
    """(tiles per CTA, images per 128-row box) of a call whose iteration lattice is lat = (D, H, W) x n, by the rules of
    conv_igemm_impl: the box is filled w, h, d, then batch; the grid has min(m-tiles, SMs / (n-tiles x phases)) CTAs."""
    rem, tiles = 128, 1
    for e in (lat[2], lat[1], lat[0]):
        b = min(_pow2_floor(e), rem)
        rem //= b
        tiles *= -(-e // b)
    m_tiles = tiles * -(-n // rem)
    if bn is None:
        bn = min((128, 64, 32), key=lambda b: (-(-n_pad // b) * b, -b))
    gx = min(m_tiles, max(1, torch.cuda.get_device_properties(0).multi_processor_count // (-(-n_pad // bn) * phases)))
    return -(-m_tiles // gx), rem


def batch_for(lat, n_pad, phases, tiles, bn=None):
    """The smallest batch whose CTAs hold `tiles` tiles, and the largest batch slice (whole boxes) at one tile per CTA."""
    n = next(n for n in range(1, 1 << 14) if launch(lat, n, n_pad, phases, bn)[0] == tiles)
    per_box = launch(lat, 1, n_pad, phases, bn)[1]
    one = max(s for s in range(per_box, n + per_box, per_box) if launch(lat, s, n_pad, phases, bn)[0] == 1)
    return n, one


def fwd_lattice(case):
    _, _, s, _, transposed, _, _, _, _, _ = case
    o = E.out_extent(case)
    return tuple(-(-e // ss) for e, ss in zip(o, s)) if transposed else o


def sliced(n, step):
    return [(b, min(n, b + step)) for b in range(0, n, step)]


@pytest.mark.parametrize('tiles', TILES_PER_CTA)
@pytest.mark.parametrize('case', CASES, ids=E.case_id)
def test_multi_tile_ctas_match_fp64_and_single_tile_ctas(L, mode, case, tiles):  # noqa: F811
    """Forward with bias and leaky relu, accumulate 1 and 2, split_k 3 and the fused activation-gradient dgrad against
    ref_conv; the forward and the fused dgrad equal the one-tile-per-CTA slices bit for bit."""
    kind, k, s, p, transposed, ci_ref, ci_int, cmap, co, ext = case
    ke = E.eff_kernel(kind, k)
    taps = ke[0] * ke[1] * ke[2]
    oext = E.out_extent(case)
    sp = s[0] * s[1] * s[2]
    w = E.rnd(*k, ci_ref, co, seed=1, scale=(k[0] * k[1] * k[2] * ci_ref) ** -0.5)
    bias = E.rnd(co, seed=2, scale=0.3)
    wp, n_pad, kc = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_FWD, ci_int=ci_int)
    wpd, n_pad_d, kc_d = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_DGRAD, ci_int=ci_int)
    n, one = batch_for(fwd_lattice(case), n_pad, sp if transposed else 1, tiles)
    ck = E.Checks('%s n=%d' % (E.case_id(case), n))
    wf, wd = E.unpack(wp, taps, n_pad, kc, co, ci_int), E.unpack(wpd, taps, n_pad_d, kc_d, ci_int, co)
    g, gt = L.geom(ke, s, p, transposed), L.geom(ke, s, p, not transposed)
    kf = taps * ci_int / (sp if transposed else 1)
    kd = taps * co / (1 if transposed else sp)

    # ---- forward
    x = E.act_input(n, ext, ci_int, None, seed=3)
    pre = E.ref_conv(E.tf32(x, mode)[..., :ci_int].double(), wf, ke, s, p, transposed, oext)
    b64 = bias.double()
    out = E.out_buf(n, oext, co)
    L.conv_igemm(L.tensor_view(x, ci_int), g, wp, n_pad, kc, L.tensor_view(out, co, E.OFF), bias, L.ACT_LRELU, E.ALPHA)
    ck.close('fwd lrelu', 'fwd', out[..., E.OFF:E.OFF + co], E.act_ref(pre + b64, L.ACT_LRELU), kf)
    ck.untouched('fwd lrelu', out, co)
    parts = E.out_buf(n, oext, co)
    for b0, b1 in sliced(n, one):
        L.conv_igemm(L.tensor_view(x[b0:b1], ci_int), g, wp, n_pad, kc, L.tensor_view(parts[b0:b1], co, E.OFF), bias,
                     L.ACT_LRELU, E.ALPHA)
    prev = E.rnd(n, *oext, co, seed=4)
    acc1 = E.out_buf(n, oext, co)
    acc1[..., E.OFF:E.OFF + co] = prev
    L.conv_igemm(L.tensor_view(x, ci_int), g, wp, n_pad, kc, L.tensor_view(acc1, co, E.OFF), None, L.ACT_NONE, 0.0, 1, 1)
    ck.close('fwd accumulate 1', 'fwd_acc', acc1[..., E.OFF:E.OFF + co], prev.double() + pre, kf)
    acc2 = E.out_buf(n, oext, co)
    acc2[..., E.OFF:E.OFF + co] = prev
    L.conv_igemm(L.tensor_view(x, ci_int), g, wp, n_pad, kc, L.tensor_view(acc2, co, E.OFF), bias, L.ACT_TANH, 0.0, 1, 2)
    ck.close('fwd accumulate 2 + bias + tanh', 'fwd_sigmoid_tanh', acc2[..., E.OFF:E.OFF + co],
             torch.tanh(prev.double() + pre + b64), kf, fast_math=True)
    split = E.out_buf(n, oext, co)
    split[..., E.OFF:E.OFF + co] = 0.0
    L.conv_igemm(L.tensor_view(x, ci_int), g, wp, n_pad, kc, L.tensor_view(split, co, E.OFF), bias, L.ACT_NONE, 0.0, 3)
    ck.close('fwd split_k 3', 'fwd_split', split[..., E.OFF:E.OFF + co], pre + b64, kf)
    ck.untouched('fwd split_k 3', split, co)

    # ---- fused activation-gradient dgrad, with addend
    dy = E.act_input(n, oext, (co + 3) // 4 * 4, None, seed=5)
    dy[..., co:] = NAN
    dref = E.ref_conv(E.tf32(dy, mode)[..., :co].double(), wd, ke, s, p, not transposed, ext)
    y = E.act_output(L.ACT_LRELU, (n,) + tuple(ext) + (ci_int,), seed=6)
    add = E.rnd(n, *ext, ci_int, seed=7)
    dx = torch.full_like(add, NAN)
    L.conv_igemm_actgrad(L.tensor_view(dy, co), gt, wpd, n_pad_d, kc_d, L.tensor_view(dx, ci_int), y.data_ptr(), add.data_ptr(),
                         L.ACT_LRELU, E.ALPHA)
    ck.close('actgrad lrelu + addend', 'actgrad', dx, (dref + add.double()) * E.act_deriv(y, L.ACT_LRELU), kd)
    dparts = torch.full_like(add, NAN)
    for b0, b1 in sliced(n, one):
        L.conv_igemm_actgrad(L.tensor_view(dy[b0:b1], co), gt, wpd, n_pad_d, kc_d, L.tensor_view(dparts[b0:b1], ci_int),
                             y[b0:b1].data_ptr(), add[b0:b1].data_ptr(), L.ACT_LRELU, E.ALPHA)
    ck.done()
    assert torch.equal(out.view(torch.int32), parts.view(torch.int32)), 'forward: the tiles of a multi-tile CTA differ'
    assert torch.equal(dx.view(torch.int32), dparts.view(torch.int32)), 'fused dgrad: the tiles of a multi-tile CTA differ'


@pytest.mark.parametrize('tiles', TILES_PER_CTA)
def test_multi_tile_conv_lstm_matches_fp64_and_single_tile_ctas(L, mode, tiles):  # noqa: F811
    """vp_conv_lstm_fwd at the long-K gate convolution (5x5 over 264 channels, F = 128: 225 k-chunks per tile, four
    128-column tiles) against fp64 as tests/test_gpu_conv_lstm.py checks it, and bit for bit against one-tile-per-CTA
    slices."""
    case = _lstm_case(8, 128)
    _, k, s, p, _, _, ci, _, co, ext = case
    F, hw = co // 4, ext[1]
    n, one = batch_for(ext, co, 1, tiles, bn=128)
    x = E.act_input(n, ext, ci, None, seed=1)
    w = E.rnd(5, 5, ci, co, seed=2, scale=0.03)
    bias = E.rnd(co, seed=3, scale=0.5)
    c_prev = E.rnd(n, hw, hw, F, seed=4)
    nat, n_pad, kc = L.pack_weights(w, k, ci, co, PLAIN, L.WLAYOUT_FWD)
    wp, _, _ = L.pack_weights(w, k, ci, co, PLAIN, L.WLAYOUT_FWD | L.WLAYOUT_GATES)
    g = L.geom(k, s, p)

    def run(b0, b1, z, c_new, h):
        L.conv_lstm_fwd(L.tensor_view(x[b0:b1].view(b1 - b0, hw, hw, -1), ci), g, wp, n_pad, kc, z[b0:b1], bias,
                        c_prev[b0:b1], c_new[b0:b1], [(h[b0:b1].data_ptr(), F)])

    bufs = [tuple(torch.full((n, hw, hw, c), NAN, device='cuda') for c in (co, F, F)) for _ in range(2)]
    run(0, n, *bufs[0])
    for b0, b1 in sliced(n, one):
        run(b0, b1, *bufs[1])
    z, c_new, h = bufs[0]
    W = E.unpack(nat, 25, n_pad, kc, co, ci)
    xq = E.tf32(x[..., :ci], mode).double()
    ref = E.ref_conv(xq, W, k, s, p, False, ext).view(n, hw, hw, co) + bias.double()
    scale = E.ref_conv(xq.abs(), W.abs(), k, s, p, False, ext).max()
    c_ref, h_ref = _cell64(z.double(), c_prev.double())
    errs = torch.stack([(z.double() - ref).abs().max() / scale, (c_new.double() - c_ref).abs().max(),
                        (h.double() - h_ref).abs().max()]).tolist()
    assert errs[0] <= 5e-6 and errs[1] <= 2e-5 and errs[2] <= 2e-5, (n, errs)
    for a, b in zip(bufs[0], bufs[1]):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), 'ConvLSTM: the tiles of a multi-tile CTA differ'
