"""Every form of the weight gradient (vp_conv_wgrad_in_form, lib.conv_wgrad_forms) against an fp64 reference and bit for
bit against the form the call's shape selects (vp_conv_wgrad).  A form only decides which CTA computes which (row blocks,
column tile, pixel-range split); every dW element stays the same chain of 8-pixel MMAs in pixel order, so every form
must give the same bits.  Operands are random TF32 values (exact products), the channels outside the views are NaN, and
the padding rows and columns of the packed dW must stay zero.  The stage cases give 1, 2, 3 and 11 stages per CTA (the
mainloop is unrolled by two and its ring holds at most 8 stages), with one pixel-range split and with several."""
import pytest
import torch

gpu = pytest.mark.gpu
NAN = float('nan')

# (k, s, p, transposed, ci, co, input extent (d, h, w), batch)
CASES = [
    ((1, 6, 6), (1, 2, 2), (0, 2, 2), False, 32, 32, (1, 32, 32), 4),      # 36 taps, strided (h0)
    ((1, 6, 6), (1, 2, 2), (0, 2, 2), True, 40, 24, (1, 8, 8), 3),         # transposed
    ((4, 4, 4), (1, 2, 2), (1, 1, 1), False, 32, 64, (5, 16, 16), 2),      # 3-D discriminator geometry
    ((1, 3, 3), (1, 1, 1), (0, 1, 1), False, 32, 3, (1, 16, 16), 3),       # co = 3
    ((1, 3, 3), (1, 1, 1), (0, 1, 1), False, 60, 8, (1, 9, 7), 5),         # co = 8, partial tiles
    ((1, 5, 5), (1, 1, 1), (0, 2, 2), False, 72, 264, (1, 8, 8), 2),       # n_tiles > 1 in every form
]


def case_id(c):
    k, s, p, t, ci, co, ext, n = c
    return 'k%s_s%s_%sci%d_co%d_%s_n%d' % (''.join(map(str, k)), ''.join(map(str, s)), 'T' if t else '', ci, co,
                                           'x'.join(map(str, ext)), n)


def out_extent(k, s, p, transposed, ext):
    if transposed:
        return tuple((i - 1) * ss - 2 * pp + kk for i, ss, pp, kk in zip(ext, s, p, k))
    return tuple((i + 2 * pp - kk) // ss + 1 for i, ss, pp, kk in zip(ext, s, p, k))


@pytest.fixture(scope='module')
def L():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from video_prediction_b200 import lib
    lib.lib()
    return lib


def tf32(t):
    return (t.view(torch.int32) & -8192).view(torch.float32)


def gather(src, lattice, s, r, p):
    """src [n, D, H, W, C] read at s * o + r - p for o over `lattice` (d, h, w); zero outside src."""
    out = src
    for dim, (size, ss, rr, pp) in enumerate(zip(lattice, s, r, p)):
        idx = torch.arange(size, device=src.device) * ss + rr - pp
        ok = (idx >= 0) & (idx < src.shape[dim + 1])
        out = out.index_select(dim + 1, idx.clamp(0, src.shape[dim + 1] - 1))
        shape = [1] * out.dim()
        shape[dim + 1] = size
        out = out * ok.view(shape).to(out.dtype)
    return out


def reference(case, x, dy):
    """fp64 dW [taps][co][ci]: conv sum_o dy[o] x[s o + r - p]; transposed sum_i dy[s i + r - p] x[i]."""
    k, s, p, transposed, ci, co, ext, n = case
    xd, dyd = x[..., :ci].double(), dy[..., :co].double()
    out = []
    for rd in range(k[0]):
        for rh in range(k[1]):
            for rw in range(k[2]):
                r = (rd, rh, rw)
                if transposed:
                    out.append(torch.einsum('ndhwo,ndhwi->oi', gather(dyd, ext, s, r, p), xd))
                else:
                    out.append(torch.einsum('ndhwo,ndhwi->oi', dyd, gather(xd, dyd.shape[1:4], s, r, p)))
    return torch.stack(out)


def operands(case, seed):
    k, s, p, transposed, ci, co, ext, n = case
    oext = out_extent(k, s, p, transposed, ext)
    gen = torch.Generator().manual_seed(seed)
    x = torch.full((n,) + tuple(ext) + (ci + 4,), NAN)
    dy = torch.full((n,) + tuple(oext) + ((co + 3) // 4 * 4 + 4,), NAN)
    x[..., :ci] = tf32(torch.randn(x[..., :ci].shape, generator=gen))
    dy[..., :co] = tf32(torch.randn(dy[..., :co].shape, generator=gen))
    return x.cuda(), dy.cuda()


def run(L, case, x, dy, split, form=None):
    k, s, p, transposed, ci, co, ext, n = case
    n_pad, kc = L.choose_n_pad(co), (ci + 31) // 32
    dw = torch.zeros(k[0] * k[1] * k[2], n_pad, kc * 32, device='cuda')
    args = (L.tensor_view(x, ci), L.tensor_view(dy, co), L.geom(k, s, p, transposed), dw, n_pad, kc, split)
    if form is None:
        L.conv_wgrad(*args)
    else:
        L.conv_wgrad_in_form(*args, form)
    return dw


def check_against_reference(case, dw, ref, where):
    k, s, p, transposed, ci, co, ext, n = case
    got = dw[:, :co, :ci].double()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 1e-5 * scale, '%s: max |err| %g, max |ref| %g' % (where, err, scale)
    pad = dw.clone()
    pad[:, :co, :ci] = 0
    assert not pad.any().item(), where + ': padding rows / columns written'


@gpu
@pytest.mark.parametrize('case', CASES, ids=case_id)
def test_every_form_against_fp64_and_bit_for_bit(L, case):
    x, dy = operands(case, 1)
    ref = reference(case, x.cpu(), dy.cpu()).cuda()
    for split in (0, 1, 3):
        base = run(L, case, x, dy, split)
        check_against_reference(case, base, ref, 'default form, split %d' % split)
        for f, (blocks, bn) in enumerate(L.conv_wgrad_forms()):
            dw = run(L, case, x, dy, split, f)
            where = 'form %d (%d blocks x %d columns), split %d' % (f, blocks, bn, split)
            check_against_reference(case, dw, ref, where)
            assert torch.equal(dw, base), where + ': bits differ from the default form'


# 8x8 images are one 64-pixel tile each, so the batch is the pixel-tile count: (batch, split_k) -> stages per CTA
STAGES = [(1, 1), (2, 1), (3, 1), (11, 1), (8, 2), (12, 3), (22, 2), (9, 2)]


@gpu
@pytest.mark.parametrize('tiles,split', STAGES, ids=['t%d_s%d' % ts for ts in STAGES])
def test_stage_counts_and_ring_wrap(L, tiles, split):
    case = ((1, 3, 3), (1, 1, 1), (0, 1, 1), False, 40, 48, (1, 8, 8), tiles)
    x, dy = operands(case, 2)
    ref = reference(case, x.cpu(), dy.cpu()).cuda()
    base = run(L, case, x, dy, split)
    check_against_reference(case, base, ref, 'default form')
    for f, (blocks, bn) in enumerate(L.conv_wgrad_forms()):
        dw = run(L, case, x, dy, split, f)
        where = 'form %d (%d blocks x %d columns)' % (f, blocks, bn)
        check_against_reference(case, dw, ref, where)
        assert torch.equal(dw, base), where + ': bits differ from the default form'


@gpu
def test_form_query_matches_the_call(L):
    """conv_wgrad_form reports a form that exists and the split count of the layer's rule."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    forms = L.conv_wgrad_forms()
    for case in CASES:
        k, s, p, transposed, ci, co, ext, n = case
        oext = out_extent(k, s, p, transposed, ext)
        f, ctas, splits, stages = L.conv_wgrad_form(L.geom(k, s, p, transposed), (n,) + tuple(ext) + (ci,),
                                                    (n,) + tuple(oext) + (co,), L.choose_n_pad(co), (ci + 31) // 32, sms, 0)
        assert 0 <= f < len(forms) and ctas >= splits >= 1 and stages >= 1
