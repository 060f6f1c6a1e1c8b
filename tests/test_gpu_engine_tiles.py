"""Every tile form of the engine's forward / dgrad kernel (igemm_fwd_kernel<kRows, BN>) at the cfg2 calls that select it.

conv_igemm_impl picks, from the call's shape alone, a tile of 128 or 64 output pixels and BN GEMM columns
(lib.conv_igemm_forms lists them, lib.conv_igemm_form gives a call's).  For every form, the first cfg2 call below that
selects it runs the forward epilogues (bias + leaky relu, accumulate 1, accumulate 2 + bias + leaky relu) and the fused
activation-gradient epilogue (with and without addend) on that call's operands, against the fp64 reference of
tests/test_gpu_engine.py with its tolerances.  The list holds a strided conv and transposed (phase-split) dgrads, which are
checked whatever form they select.  Each output element is one chain of K = 8 MMAs in tap / chunk order in every form, so a
call whose batch slices select another form than the full batch must give the same bits."""
import pytest
import torch

import test_gpu_engine as E
from test_gpu_engine import L, mode  # noqa: F401  (fixtures of the engine check)
from test_gpu_engine import PLAIN, POOLED, S1, S2, UPSAMPLED, _case

pytestmark = pytest.mark.gpu
NAN = float('nan')

# (case, batch, direction) of cfg2 calls (B = 16: generator convs see 2B images, the video discriminator B clips of 10
# frames): 'fwd' runs the case's convolution, 'dgrad' its input gradient (the flipped geometry, DGRAD pack)
CALLS = [
    (_case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, 72, 128, (1, 32, 32)), 32, 'fwd'),     # lstm_h0 gates
    (_case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, 72, 128, (1, 32, 32)), 32, 'dgrad'),   # n_pad 80
    (_case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, 136, 256, (1, 16, 16)), 32, 'dgrad'),  # n_pad 144
    (_case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, 264, 512, (1, 8, 8)), 32, 'dgrad'),    # n_pad 288
    (_case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, 136, 256, (1, 16, 16)), 32, 'fwd'),
    (_case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, 264, 512, (1, 8, 8)), 32, 'fwd'),
    (_case(POOLED, (1, 3, 3), S2, (0, 1, 1), False, 72, 128, (1, 16, 16)), 32, 'fwd'),    # strided (h2)
    (_case(POOLED, (1, 3, 3), S2, (0, 1, 1), False, 72, 128, (1, 16, 16)), 32, 'dgrad'),  # phase-split
    (_case(UPSAMPLED, (1, 3, 3), S2, (0, 2, 2), True, 136, 64, (1, 8, 8)), 32, 'fwd'),    # phase-split (h3)
    (_case(UPSAMPLED, (1, 3, 3), S2, (0, 2, 2), True, 136, 64, (1, 8, 8)), 32, 'dgrad'),  # n_pad 144, strided
    (_case(UPSAMPLED, (1, 3, 3), S2, (0, 2, 2), True, 72, 32, (1, 32, 32)), 32, 'dgrad'),  # n_pad 80
    (_case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 32, 32, (1, 64, 64)), 32, 'fwd'),
    (_case(PLAIN, (3, 3, 3), S1, (1, 1, 1), False, 64, 64, (9, 32, 32)), 16, 'fwd'),
    (_case(PLAIN, (4, 4, 4), S2, (1, 1, 1), False, 64, 128, (9, 32, 32)), 16, 'dgrad'),
    (_case(PLAIN, (3, 3, 3), S1, (1, 1, 1), False, 256, 256, (4, 8, 8)), 16, 'fwd'),
]


class Call(object):
    """Operands, packs and fp64 pre-activation reference of one engine call; the output extent is `oext`, the output
    channels `co`, K the products summed into one output element."""

    def __init__(self, L, mode, case, n, direction):  # noqa: F811
        kind, k, s, p, transposed, ci_ref, ci_int, cmap, co, ext = case
        ke = E.eff_kernel(kind, k)
        taps = ke[0] * ke[1] * ke[2]
        sp = s[0] * s[1] * s[2]
        w = E.rnd(*k, ci_ref, co, seed=1, scale=(k[0] * k[1] * k[2] * ci_ref) ** -0.5)
        cm = None if cmap is None else torch.tensor(cmap, dtype=torch.int32, device='cuda')
        if direction == 'fwd':
            self.wp, self.n_pad, self.kc = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_FWD, ci_int=ci_int, cmap=cm)
            wm = E.unpack(self.wp, taps, self.n_pad, self.kc, co, ci_int)
            self.g, ci, self.co, iext, self.oext, tr = L.geom(ke, s, p, transposed), ci_int, co, ext, E.out_extent(case), transposed
            self.K = taps * ci_int / (sp if transposed else 1)
        else:
            self.wp, self.n_pad, self.kc = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_DGRAD, ci_int=ci_int, cmap=cm)
            wm = E.unpack(self.wp, taps, self.n_pad, self.kc, ci_int, co)
            self.g, ci, self.co, iext, self.oext, tr = L.geom(ke, s, p, not transposed), co, ci_int, E.out_extent(case), ext, not transposed
            self.K = taps * co / (1 if transposed else sp)
        self.L, self.n, self.ci = L, n, ci
        self.x = E.act_input(n, iext, (ci + 3) // 4 * 4, cmap if direction == 'fwd' else None, seed=3)
        self.x[..., ci:] = NAN
        self.ref = E.ref_conv(E.tf32(self.x, mode)[..., :ci].double(), wm, ke, s, p, tr, self.oext)
        self.form = self.form_of(L, n)

    def form_of(self, L, n):  # noqa: F811
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        return L.conv_igemm_form(self.g, (n,) + tuple(self.oext), self.n_pad, self.kc, sms)

    def xv(self, b0=0, b1=None):
        return self.L.tensor_view(self.x[b0:b1], self.ci)


def _first_call(L, mode, form):  # noqa: F811
    for case, n, direction in CALLS:
        c = Call(L, mode, case, n, direction)
        if c.form == form:
            return c
    return None


def test_cfg2_calls_cover_every_form(L, mode):  # noqa: F811
    """Every form the rule can pick is selected by one of CALLS, so test_form_matches_fp64 checks each of them."""
    seen = {Call(L, mode, case, n, d).form for case, n, d in CALLS}
    assert set(L.conv_igemm_forms()) <= seen, (L.conv_igemm_forms(), seen)


@pytest.mark.parametrize('form', [(128, 32), (128, 64), (128, 80), (128, 128), (64, 32), (64, 64), (64, 80), (64, 128),
                                  (64, 144)], ids=lambda f: '%dx%d' % f)
def test_form_matches_fp64(L, mode, form):  # noqa: F811
    """Bias + leaky relu, accumulate 1, accumulate 2 + bias + leaky relu and the fused leaky-relu gradient with and without
    addend, on the first cfg2 call that selects `form`.  (The fast-math sigmoid / tanh epilogue, which does not depend on
    the form, is left to tests/test_gpu_engine.py: over the 0.5 M outputs of a cfg2 call its max-abs error reaches 1.3e-4.)"""
    c = _first_call(L, mode, form)
    assert c is not None, 'no call of CALLS selects %dx%d' % form
    ck = E.Checks('%dx%d' % form)
    n, co, oext = c.n, c.co, c.oext
    bias = E.rnd(co, seed=2, scale=0.3)
    b64 = bias.double()
    out = E.out_buf(n, oext, co)
    L.conv_igemm(c.xv(), c.g, c.wp, c.n_pad, c.kc, L.tensor_view(out, co, E.OFF), bias, L.ACT_LRELU, E.ALPHA)
    ck.close('fwd lrelu', 'fwd', out[..., E.OFF:E.OFF + co], E.act_ref(c.ref + b64, L.ACT_LRELU), c.K)
    ck.untouched('fwd lrelu', out, co)
    prev = E.rnd(n, *oext, co, seed=4)
    acc1 = E.out_buf(n, oext, co)
    acc1[..., E.OFF:E.OFF + co] = prev
    L.conv_igemm(c.xv(), c.g, c.wp, c.n_pad, c.kc, L.tensor_view(acc1, co, E.OFF), None, L.ACT_NONE, 0.0, 1, 1)
    ck.close('fwd accumulate 1', 'fwd_acc', acc1[..., E.OFF:E.OFF + co], prev.double() + c.ref, c.K)
    acc2 = E.out_buf(n, oext, co)
    acc2[..., E.OFF:E.OFF + co] = prev
    L.conv_igemm(c.xv(), c.g, c.wp, c.n_pad, c.kc, L.tensor_view(acc2, co, E.OFF), bias, L.ACT_LRELU, E.ALPHA, 1, 2)
    ck.close('fwd accumulate 2 + bias + lrelu', 'fwd', acc2[..., E.OFF:E.OFF + co],
             E.act_ref(prev.double() + c.ref + b64, L.ACT_LRELU), c.K)
    y = E.act_output(L.ACT_LRELU, (n,) + tuple(oext) + (co,), seed=6)
    add = E.rnd(n, *oext, co, seed=7)
    for addend in (None, add):
        dx = torch.full_like(add, NAN)
        L.conv_igemm_actgrad(c.xv(), c.g, c.wp, c.n_pad, c.kc, L.tensor_view(dx, co), y.data_ptr(),
                             0 if addend is None else addend.data_ptr(), L.ACT_LRELU, E.ALPHA)
        v = c.ref + (0.0 if addend is None else addend.double())
        ck.close('actgrad lrelu addend %d' % (addend is not None), 'actgrad', dx, v * E.act_deriv(y, L.ACT_LRELU), c.K)
    ck.done()


@pytest.mark.parametrize('i', range(len(CALLS)))
def test_strided_and_phase_split_calls_match_fp64(L, mode, i):  # noqa: F811
    """Every call of CALLS, plain output, against fp64, whatever form it selects."""
    c = Call(L, mode, *CALLS[i])
    ck = E.Checks('call %d %dx%d' % ((i,) + c.form))
    out = E.out_buf(c.n, c.oext, c.co)
    L.conv_igemm(c.xv(), c.g, c.wp, c.n_pad, c.kc, L.tensor_view(out, c.co, E.OFF))
    ck.close('conv', 'fwd', out[..., E.OFF:E.OFF + c.co], c.ref, c.K)
    ck.untouched('conv', out, c.co)
    ck.done()


def test_batch_slices_of_another_form_give_the_same_bits(L, mode):  # noqa: F811
    """A call whose full batch and whose batch slices select different forms: forward and fused dgrad are bit-identical."""
    found = 0
    for case, n, direction in CALLS:
        c = Call(L, mode, case, n, direction)
        step = next((s for s in (16, 8, 4, 2, 1) if n % s == 0 and c.form_of(L, s) != c.form), None)
        if step is None:
            continue
        found += 1
        bias = E.rnd(c.co, seed=2, scale=0.3)
        y = E.act_output(L.ACT_LRELU, (n,) + tuple(c.oext) + (c.co,), seed=6)
        add = E.rnd(n, *c.oext, c.co, seed=7)
        full, parts = E.out_buf(n, c.oext, c.co), E.out_buf(n, c.oext, c.co)
        dfull, dparts = torch.full_like(add, NAN), torch.full_like(add, NAN)
        L.conv_igemm(c.xv(), c.g, c.wp, c.n_pad, c.kc, L.tensor_view(full, c.co, E.OFF), bias, L.ACT_LRELU, E.ALPHA)
        L.conv_igemm_actgrad(c.xv(), c.g, c.wp, c.n_pad, c.kc, L.tensor_view(dfull, c.co), y.data_ptr(), add.data_ptr(),
                             L.ACT_LRELU, E.ALPHA)
        for b0 in range(0, n, step):
            b1 = b0 + step
            L.conv_igemm(c.xv(b0, b1), c.g, c.wp, c.n_pad, c.kc, L.tensor_view(parts[b0:b1], c.co, E.OFF), bias, L.ACT_LRELU,
                         E.ALPHA)
            L.conv_igemm_actgrad(c.xv(b0, b1), c.g, c.wp, c.n_pad, c.kc, L.tensor_view(dparts[b0:b1], c.co), y[b0:b1].data_ptr(),
                                 add[b0:b1].data_ptr(), L.ACT_LRELU, E.ALPHA)
        what = '%s n=%d (%dx%d) against slices of %d (%dx%d)' % ((E.case_id(case), n) + c.form + (step,) + c.form_of(L, step))
        assert torch.equal(full.view(torch.int32), parts.view(torch.int32)), 'forward: ' + what
        assert torch.equal(dfull.view(torch.int32), dparts.view(torch.int32)), 'fused dgrad: ' + what
    assert found, 'no call of CALLS changes form between its batch and a batch slice'
