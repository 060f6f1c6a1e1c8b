"""The tensor-core convolution engine (csrc/igemm.cu: vp_conv_igemm, vp_conv_igemm_actgrad, vp_conv_wgrad) and its weight
packing (csrc/pack.cu), at every layer geometry the model runs and at the engine's edges.

The judge is `ref_conv`, an fp64 evaluation of the geometry exactly as include/vp_b200.h defines it (vp_conv_geom), proven
against torch's convolutions by a CPU test.  The engine is fed the operands the tensor core actually reads: activations
quantised the way the tensor core quantises fp32 operands (identified by a probe, not assumed) and the packed weight
buffer itself, read back tap by tap.  What is left between the engine and the reference is fp32 accumulation order, so the
tolerances are a few times that floor; packing is checked on its own against effective kernels built here.

Every call writes into a channel slice of a wider buffer whose other channels hold NaN (they must come back untouched), reads
an input whose channels outside the view hold NaN (they must not be read), and overwrites an in-view output prefilled with
NaN unless it accumulates.  In-view padding channels that the channel map sends to -1 stay zero, as in the model."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu           # everything but the reference's own tests needs the H100
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
NAN = float('nan')


# ------------------------------------------------------------------ fp64 reference of vp_conv_geom
def _tap_slices(t, k, s, p, n_out):
    """For every tap r = (rd, rh, rw) (tap index (rd*kh + rh)*kw + rw): the view of t [N, D, H, W, C] at s*o + r - p for
    o < n_out on each axis, zero outside t."""
    hi = [max(0, (kk - 1) + ss * (o - 1) - pp - (i - 1)) for kk, ss, pp, o, i in zip(k, s, p, n_out, t.shape[1:4])]
    tp = F.pad(t, (0, 0, p[2], hi[2], p[1], hi[1], p[0], hi[0]))
    out = []
    for rd in range(k[0]):
        for rh in range(k[1]):
            for rw in range(k[2]):
                out.append(tp[:, rd:rd + s[0] * (n_out[0] - 1) + 1:s[0], rh:rh + s[1] * (n_out[1] - 1) + 1:s[1],
                              rw:rw + s[2] * (n_out[2] - 1) + 1:s[2]])
    return out


def ref_conv(x, w, k, s, p, transposed, out_sp):
    """x [N, D, H, W, Ci], w [taps, Ci, Co] (the effective tap matrices), out_sp = (OD, OH, OW).
    transposed == 0: out[o] = sum_r x[s*o + r - p] @ w[r];  transposed == 1: x[o] @ w[r] is added into out[s*o + r - p].
    Reads and writes outside the tensors are zero / dropped."""
    n, co = x.shape[0], w.shape[-1]
    if not transposed:
        out = x.new_zeros(n, *out_sp, co)
        for r, sl in enumerate(_tap_slices(x, k, s, p, out_sp)):
            out += sl @ w[r]
        return out
    insp = x.shape[1:4]
    # padded output index s*o + r covers [0, s*(In-1) + k); output index i sits at i + p
    ext = [max(ss * (i - 1) + kk, pp + o) for ss, i, kk, pp, o in zip(s, insp, k, p, out_sp)]
    buf = x.new_zeros(n, *ext, co)
    r = 0
    for rd in range(k[0]):
        for rh in range(k[1]):
            for rw in range(k[2]):
                buf[:, rd:rd + s[0] * (insp[0] - 1) + 1:s[0], rh:rh + s[1] * (insp[1] - 1) + 1:s[1],
                    rw:rw + s[2] * (insp[2] - 1) + 1:s[2]] += x @ w[r]
                r += 1
    return buf[:, p[0]:p[0] + out_sp[0], p[1]:p[1] + out_sp[1], p[2]:p[2] + out_sp[2]].contiguous()


def ref_wgrad(x, dy, k, s, p, transposed):
    """dW[r] [Ci, Co] = d <dy, ref_conv(x, W)> / d W[r]."""
    ci, co = x.shape[-1], dy.shape[-1]
    if not transposed:      # sum_o x[s*o + r - p]^T dy[o]
        return torch.stack([sl.reshape(-1, ci).t() @ dy.reshape(-1, co) for sl in _tap_slices(x, k, s, p, dy.shape[1:4])])
    # sum_o x[o]^T dy[s*o + r - p]
    return torch.stack([x.reshape(-1, ci).t() @ sl.reshape(-1, co) for sl in _tap_slices(dy, k, s, p, x.shape[1:4])])


def _torch_weight(w, k, transposed):
    wk = w.reshape(*k, w.shape[1], w.shape[2])                 # [kd, kh, kw, Ci, Co]
    return wk.permute(3, 4, 0, 1, 2) if transposed else wk.permute(4, 3, 0, 1, 2)


# ------------------------------------------------------------------ layer geometries
def concat(*valid):
    """(ci_ref, ci_int, cmap) of a concat buffer whose segments hold `valid` channels each, every segment padded to a
    multiple of 4 channels; cmap is None when it is the identity."""
    cmap, ref = [], 0
    for v in valid:
        a = (v + 3) // 4 * 4
        cmap += list(range(ref, ref + v)) + [-1] * (a - v)
        ref += v
    ident = cmap == list(range(len(cmap)))
    return ref, len(cmap), None if ident else tuple(cmap)


PLAIN, POOLED, UPSAMPLED = 0, 1, 2
S1, S2, S222 = (1, 1, 1), (1, 2, 2), (2, 2, 2)


def _case(kind, k, s, p, transposed, ch, co, ext):
    ci_ref, ci_int, cmap = concat(*ch) if isinstance(ch, tuple) else (ch, ch, None)
    return (kind, k, s, p, transposed, ci_ref, ci_int, cmap, co, ext)


# (kind, kernel, stride, pad before, transposed, ci_ref, ci_int, cmap, co, input extent (D, H, W)) of every convolution of
# the model: generator encoder/decoder (cfg2: 64x64x3, ngf 32, nz 8), ConvLSTM gate convs, output convs (CDNA and flow),
# posterior encoder (nef 64), video discriminator (ndf 32, clip 10) and image discriminator.
MODEL_CASES = [
    # generator: conv_pool2d (image | first image | z), ConvLSTM gates (x | z | h), upsample_conv2d (x | skip | z)
    _case(POOLED, (1, 5, 5), S2, (0, 2, 2), False, (3, 3, 8), 32, (1, 64, 64)),
    _case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, 72, 128, (1, 32, 32)),
    _case(POOLED, (1, 3, 3), S2, (0, 1, 1), False, 40, 64, (1, 32, 32)),
    _case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, 136, 256, (1, 16, 16)),
    _case(POOLED, (1, 3, 3), S2, (0, 1, 1), False, 72, 128, (1, 16, 16)),
    _case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, 264, 512, (1, 8, 8)),
    _case(UPSAMPLED, (1, 3, 3), S2, (0, 2, 2), True, 136, 64, (1, 8, 8)),
    _case(UPSAMPLED, (1, 3, 3), S2, (0, 2, 2), True, 136, 32, (1, 16, 16)),
    _case(UPSAMPLED, (1, 3, 3), S2, (0, 2, 2), True, 72, 32, (1, 32, 32)),
    # output convs: h_scratch / h_masks / h_flow, scratch_image (co 3), masks (hm | 7 layers of 3 colours, co 7), flows (co 8)
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 32, 32, (1, 64, 64)),
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 32, 3, (1, 64, 64)),
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, (32, 3, 3, 3, 3, 3, 3, 3), 7, (1, 64, 64)),
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 32, 8, (1, 64, 64)),
    # posterior encoder: 4x4 stride-2 convs over (frame t | frame t+1)
    _case(PLAIN, (1, 4, 4), S2, (0, 1, 1), False, (3, 3), 64, (1, 64, 64)),
    _case(PLAIN, (1, 4, 4), S2, (0, 1, 1), False, 64, 128, (1, 32, 32)),
    _case(PLAIN, (1, 4, 4), S2, (0, 1, 1), False, 128, 256, (1, 16, 16)),
    # video discriminator, strides (1,1,1), (1,2,2), (2,2,2)
    _case(PLAIN, (3, 3, 3), S1, (1, 1, 1), False, (3,), 32, (10, 64, 64)),
    _case(PLAIN, (4, 4, 4), S2, (1, 1, 1), False, 32, 64, (10, 64, 64)),
    _case(PLAIN, (3, 3, 3), S1, (1, 1, 1), False, 64, 64, (9, 32, 32)),
    _case(PLAIN, (4, 4, 4), S2, (1, 1, 1), False, 64, 128, (9, 32, 32)),
    _case(PLAIN, (3, 3, 3), S1, (1, 1, 1), False, 128, 128, (8, 16, 16)),
    _case(PLAIN, (4, 4, 4), S222, (1, 1, 1), False, 128, 256, (8, 16, 16)),
    _case(PLAIN, (3, 3, 3), S1, (1, 1, 1), False, 256, 256, (4, 8, 8)),
    # image discriminator (one frame per video)
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, (3,), 32, (1, 64, 64)),
    _case(PLAIN, (1, 4, 4), S2, (0, 1, 1), False, 32, 64, (1, 64, 64)),
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 64, 64, (1, 32, 32)),
    _case(PLAIN, (1, 4, 4), S2, (0, 1, 1), False, 64, 128, (1, 32, 32)),
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 128, 128, (1, 16, 16)),
    _case(PLAIN, (1, 4, 4), S2, (0, 1, 1), False, 128, 256, (1, 16, 16)),
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 256, 256, (1, 8, 8)),
]

# Engine edges the model does not reach: odd extents under stride 2 on every axis (parity lattices of unequal size), a
# batch that is not a multiple of the box's batch depth, every k_tail (ci mod 32 in 1..8, 17..24, 25..32 and 9..16 come
# from the model) and kc from 1 to 9, and every N tile choice: BN wider than n_pad (co 3, 7, 16), BN 64 (co 48), BN 32 over
# several tiles (80, 144), choose_n_pad above 256 (264 -> 288) and BN 128 (512).
EDGE_CASES = [
    _case(PLAIN, (4, 4, 4), S222, (1, 1, 1), False, 24, 48, (9, 13, 11)),
    _case(PLAIN, (1, 4, 4), S2, (0, 1, 1), False, 40, 80, (1, 13, 11)),
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 56, 16, (1, 4, 4)),
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 8, 3, (1, 12, 10)),
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 24, 7, (1, 9, 7)),
    _case(PLAIN, (1, 3, 3), S1, (0, 1, 1), False, 56, 144, (1, 8, 8)),
    _case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, 264, 264, (1, 6, 6)),
    _case(POOLED, (1, 3, 3), S2, (0, 1, 1), False, 136, 80, (1, 9, 11)),
    _case(UPSAMPLED, (1, 3, 3), S2, (0, 2, 2), True, 40, 48, (1, 5, 7)),
    _case(PLAIN, (3, 3, 3), S1, (1, 1, 1), False, 72, 512, (3, 4, 4)),
]
BATCH = {(1, 4, 4): 7}          # N not a multiple of the box's batch depth (4x4 planes: 8 planes per 128-row box)


def eff_kernel(kind, k):
    return k if kind == PLAIN else ((1, k[1] + 1, k[2] + 1) if kind == POOLED else (1, k[1] + 3, k[2] + 3))


def out_extent(case):
    kind, k, s, p, transposed, _, _, _, _, ext = case
    ke = eff_kernel(kind, k)
    if transposed:
        return tuple((i - 1) * ss - 2 * pp + kk for i, ss, pp, kk in zip(ext, s, p, ke))
    return tuple((i + 2 * pp - kk) // ss + 1 for i, ss, pp, kk in zip(ext, s, p, ke))


def case_id(c):
    kind, k, s, p, t, ci_ref, ci_int, cmap, co, ext = c
    return '%s_k%s_s%s_%s%d-%d_co%d_%s' % ('PMU'[kind], ''.join(map(str, k)), ''.join(map(str, s)), 'T' if t else '', ci_ref,
                                            ci_int, co, 'x'.join(map(str, ext)))


# ------------------------------------------------------------------ CPU: the reference itself
@pytest.mark.parametrize('seed', range(6))
def test_reference_geometry_matches_torch_convolutions(seed):
    """ref_conv and ref_wgrad against F.conv3d / F.conv_transpose3d / autograd in fp64 on small random geometries, including
    outputs larger than the symmetric padding gives (the SAME convolutions of the model pad more at the end)."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda lo, hi: int(torch.randint(lo, hi + 1, (1,), generator=g))
    k = (ri(1, 3), ri(1, 4), ri(1, 5))
    s = (ri(1, 2), ri(1, 2), ri(1, 3))
    p = tuple(ri(0, kk - 1) for kk in k)
    ins = (ri(k[0], 5), ri(k[1], 8), ri(k[2], 9))
    n, ci, co = 2, ri(1, 5), ri(1, 6)
    x = torch.randn(n, *ins, ci, dtype=torch.float64, generator=g)
    w = torch.randn(k[0] * k[1] * k[2], ci, co, dtype=torch.float64, generator=g)
    xn = x.permute(0, 4, 1, 2, 3)
    # forward, symmetric padding
    ref = F.conv3d(xn, _torch_weight(w, k, False), stride=s, padding=p).permute(0, 2, 3, 4, 1)
    got = ref_conv(x, w, k, s, p, False, ref.shape[1:4])
    assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12)
    # forward, one extra output on each axis (reads past the end are zero)
    extra = tuple(o + 1 for o in ref.shape[1:4])
    hi = [ss * (o - 1) + kk - pp - i for ss, o, kk, pp, i in zip(s, extra, k, p, ins)]
    ref2 = F.conv3d(F.pad(xn, (p[2], max(hi[2], 0), p[1], max(hi[1], 0), p[0], max(hi[0], 0))), _torch_weight(w, k, False),
                    stride=s).permute(0, 2, 3, 4, 1)[:, :extra[0], :extra[1], :extra[2]]
    assert torch.allclose(ref_conv(x, w, k, s, p, False, extra), ref2, rtol=1e-12, atol=1e-12)
    # transposed, with and without output padding
    for op in (0, 1):
        opad = tuple(min(op, ss - 1) for ss in s)
        w_t = torch.randn(k[0] * k[1] * k[2], ci, co, dtype=torch.float64, generator=g)
        reft = F.conv_transpose3d(xn, _torch_weight(w_t, k, True), stride=s, padding=p, output_padding=opad).permute(0, 2, 3, 4, 1)
        assert torch.allclose(ref_conv(x, w_t, k, s, p, True, reft.shape[1:4]), reft, rtol=1e-12, atol=1e-12)
    # the weight gradient of both directions is the gradient of <dy, conv(x, W)>
    for transposed in (False, True):
        oshape = ref.shape[1:4] if not transposed else reft.shape[1:4]
        wr = torch.zeros_like(w, requires_grad=True)
        dy = torch.randn(n, *oshape, co, dtype=torch.float64, generator=g)
        (gw,) = torch.autograd.grad((ref_conv(x, wr, k, s, p, transposed, oshape) * dy).sum(), wr)
        assert torch.allclose(ref_wgrad(x, dy, k, s, p, transposed), gw, rtol=1e-12, atol=1e-12)


def test_geometry_table_is_consistent():
    """Every case has a positive output extent and a channel map of ci_int entries that names each reference channel once."""
    for c in MODEL_CASES + EDGE_CASES:
        kind, k, s, p, t, ci_ref, ci_int, cmap, co, ext = c
        assert all(o > 0 for o in out_extent(c)), c
        assert ci_int % 4 == 0 and ci_int >= ci_ref
        if cmap is not None:
            assert len(cmap) == ci_int and sorted(v for v in cmap if v >= 0) == list(range(ci_ref))


# ------------------------------------------------------------------ GPU: the engine against the reference
# Operand-exact comparisons: relative L2 error and max-abs error over max|ref|.  The engine and the reference read the same
# operands, so what is left is fp32 accumulation (and __expf / tanhf in the fused activations).  That floor grows with the
# number K of products summed into one output, as 2^-24 sqrt(K): a flat 1e-5 holds up to K ~ 2000 and fails the gate convs
# (K = 25 x 264 = 6600: 1.2e-5) and the first-layer weight gradient (K = 40960 pixels: 8.9e-5), so the relative L2 bound is a
# multiple of that floor.  Worst measured on an H100 80GB HBM3 (700 W) over every case of this file, beside each constant.
ACC_FLOOR = 10.0        # relative L2 <= ACC_FLOOR * 2^-24 * sqrt(K); measured worst 7.4 (first-layer wgrad, split_k 1, K = 40960);
                        # forward 2.8, dgrad and actgrad 3.6, 3xTF32 mode 2.2
MAX_ABS = 1e-4          # max-abs error <= MAX_ABS * max|ref|; measured worst 8.2e-5 (the same wgrad), forward 6.7e-5
PACK_TOL = 2e-5         # effective kernels whose TF32 rounding is exact: fp64 noise only; measured worst 0
EXACT_REL = 4 * 2.0 ** -21   # 3xTF32 on the raw fp32 operands, + the accumulation bound above: the accumulation dominates
                             # (measured worst 8.4e-6 = 2.2 floors at K = 4096, against 2^-22 for the dropped lo x lo term)
FAST_MATH_REL = 4 * 2.0 ** -21   # + for the fused sigmoid / tanh (__expf, fast tanhf): 4.2e-6 measured at K = 36 (first layer)
ALPHA = 0.2
OFF = 4                 # outputs are written into channels [OFF, OFF + c) of a wider buffer
WORST = {}


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).cuda()


def tf32(x, mode):
    """fp32 -> the TF32 value the tensor core reads ('trunc': low 13 mantissa bits dropped; 'rna': nearest, ties away)."""
    xi = x.contiguous().view(torch.int32)
    xi = ((xi + 0x1000) if mode == 'rna' else xi) & ~0x1FFF
    return xi.view(torch.float32)


@pytest.fixture(scope='module')
def L():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from video_prediction_b200 import lib
    lib.lib()
    yield lib
    if WORST:
        print('\nworst error per tolerance constant and call:')
        for k in sorted(WORST):
            print('  %-22s %.3e  %s' % (k, WORST[k][0], WORST[k][1]))


@pytest.fixture(scope='module')
def mode(L):
    """How the tensor core quantises fp32 activation operands, measured on all-positive operands (where 'trunc' and 'rna'
    differ by ~5e-4 relative) with the packed weights as the other operand."""
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(2, 8, 16, 32, generator=g) + 0.5).cuda()
    w = (torch.rand(1, 1, 1, 32, 16, generator=g) + 0.5).cuda()
    wp, n_pad, kc = L.pack_weights(w, (1, 1, 1), 32, 16, PLAIN, L.WLAYOUT_FWD)
    out = torch.zeros(2, 8, 16, 16, device='cuda')
    L.conv_igemm(L.tensor_view(x, 32), L.geom((1, 1, 1)), wp, n_pad, kc, L.tensor_view(out, 16))
    wq = wp.view(n_pad, kc * 32)[:16, :32].double().t()
    errs = {m: (out.double().reshape(-1, 16) - tf32(x, m).double().reshape(-1, 32) @ wq).abs().max().item() for m in ('trunc', 'rna')}
    best = min(errs, key=errs.get)
    assert errs[best] < 2e-5 and errs['rna' if best == 'trunc' else 'trunc'] > 10 * errs[best], errs
    return best


class Checks(object):
    """Comparisons of one case, evaluated on the device and read back with one synchronisation."""

    def __init__(self, what):
        self.what, self.errs, self.flags = what, [], []

    def close(self, name, key, got, ref, K, exact=False, fast_math=False):
        """K: products summed into one output element (per split); fast_math: the result went through sigmoid / tanh"""
        d = got.double() - ref
        floor = 2.0 ** -24 * K ** 0.5
        rel = ACC_FLOOR * floor + (EXACT_REL if exact else 0.0) + (FAST_MATH_REL if fast_math else 0.0)
        key = ('EXACT_REL/' if exact else '') + key
        self.errs.append((name, key, floor, rel, d.norm() / ref.norm().clamp_min(1e-300), d.abs().max() / ref.abs().max().clamp_min(1e-300)))

    def untouched(self, name, buf, c):
        """the channels of `buf` outside [OFF, OFF + c) still hold NaN"""
        self.flags.append((name, torch.isnan(buf[..., :OFF]).all() & torch.isnan(buf[..., OFF + c:]).all()))

    def done(self):
        vals = torch.stack([torch.stack([e[4], e[5]]) for e in self.errs]).tolist() if self.errs else []
        flags = torch.stack([f[1] for f in self.flags]).tolist() if self.flags else []
        bad = []
        for (name, key, floor, rel, _, _), (er, em) in zip(self.errs, vals):
            # recorded: the relative L2 error in units of the accumulation floor, and the max-abs error over max|ref|
            for const, v, rec, tol in (('rel L2', er, er / floor, rel), ('max-abs', em, em, MAX_ABS)):
                k = '%s/%s' % ('ACC_FLOOR' if const == 'rel L2' else 'MAX_ABS', key)
                if not (rec <= WORST.get(k, (-1.0,))[0]):
                    WORST[k] = (rec, '%s %s' % (self.what, name))
                if not v <= tol:
                    bad.append('%s: %s %.3e > %.2e' % (name, const, v, tol))
        bad += ['%s: channels outside the output view were written' % n for (n, _), ok in zip(self.flags, flags) if not ok]
        assert not bad, '%s: %s' % (self.what, '; '.join(bad))


def act_ref(v, act):
    return [lambda t: t, torch.relu, lambda t: torch.maximum(ALPHA * t, t), torch.sigmoid, torch.tanh][act](v)


def act_output(act, shape, seed):
    """A plausible output y of activation `act` (both signs for relu / lrelu)."""
    y = rnd(*shape, seed=seed)
    return torch.sigmoid(y) if act == 3 else (torch.tanh(y) if act == 4 else y)


def act_deriv(y, act):
    """act' evaluated from the activation output y, in fp64"""
    y = y.double()
    return [torch.ones_like(y), (y > 0).double(), torch.where(y > 0, 1.0, ALPHA), y * (1 - y), 1 - y * y][act]


def unpack(wp, taps, n_pad, kc, rows, cols):
    """Effective tap matrices [taps][cols][rows] (GEMM K x N, fp64) of a packed buffer whose tap rows are GEMM N."""
    return wp.view(taps, n_pad, kc * 32)[:, :rows, :cols].double().transpose(1, 2)


def act_input(n, ext, c, cmap, seed):
    """[n, D, H, W, c + 4]: channels >= c (outside the view) NaN; in-view channels that cmap sends to -1 zero."""
    t = rnd(n, *ext, c + 4, seed=seed)
    t[..., c:] = NAN
    if cmap is not None:
        t[..., [i for i, v in enumerate(cmap) if v < 0]] = 0.0
    return t


def out_buf(n, ext, c):
    return torch.full((n,) + tuple(ext) + ((c + 3) // 4 * 4 + 8,), NAN, device='cuda')


def batch_of(ext):
    return BATCH.get(ext, 1 if ext[0] > 1 and ext[1] >= 32 else 2)


@gpu
@pytest.mark.parametrize('case', MODEL_CASES + EDGE_CASES, ids=case_id)
def test_engine_matches_fp64_reference(L, mode, case):
    """Forward with bias and every activation, accumulate = 1 and 2, split-K forward, dgrad, the fused activation-gradient
    dgrad (every aux activation, with and without addend, accumulate 0 and 2) and the weight gradient at split_k 0 (auto),
    1, 2, 3, 7 of one layer geometry, against ref_conv / ref_wgrad on the operands the tensor core reads."""
    kind, k, s, p, transposed, ci_ref, ci_int, cmap, co, ext = case
    ke = eff_kernel(kind, k)
    taps = ke[0] * ke[1] * ke[2]
    oext = out_extent(case)
    n = batch_of(ext)
    ck = Checks(case_id(case))
    sp = s[0] * s[1] * s[2]
    kf = taps * ci_int / (sp if transposed else 1)          # products per output: forward
    kd = taps * co / (1 if transposed else sp)              # dgrad (the flipped geometry)
    kw = n * (ext[0] * ext[1] * ext[2] if transposed else oext[0] * oext[1] * oext[2])    # wgrad, unsplit
    cm = None if cmap is None else torch.tensor(cmap, dtype=torch.int32, device='cuda')
    w = rnd(*k, ci_ref, co, seed=1, scale=(k[0] * k[1] * k[2] * ci_ref) ** -0.5)
    bias = rnd(co, seed=2, scale=0.3)
    wp, n_pad, kc = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_FWD, ci_int=ci_int, cmap=cm)
    wpd, n_pad_d, kc_d = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_DGRAD, ci_int=ci_int, cmap=cm)
    wf, wd = unpack(wp, taps, n_pad, kc, co, ci_int), unpack(wpd, taps, n_pad_d, kc_d, ci_int, co)
    g, gt = L.geom(ke, s, p, transposed), L.geom(ke, s, p, not transposed)

    # ---- forward
    x = act_input(n, ext, ci_int, cmap, seed=3)
    xv = L.tensor_view(x, ci_int)
    pre = ref_conv(tf32(x, mode)[..., :ci_int].double(), wf, ke, s, p, transposed, oext)
    b64 = bias.double()
    for act in range(5):
        out = out_buf(n, oext, co)
        L.conv_igemm(xv, g, wp, n_pad, kc, L.tensor_view(out, co, OFF), bias, act, ALPHA)
        ck.close('fwd act %d' % act, 'fwd' if act < 3 else 'fwd_sigmoid_tanh', out[..., OFF:OFF + co], act_ref(pre + b64, act), kf,
                 fast_math=act >= 3)
        ck.untouched('fwd act %d' % act, out, co)
    prev = rnd(n, *oext, co, seed=4)
    out = out_buf(n, oext, co)
    out[..., OFF:OFF + co] = prev
    L.conv_igemm(xv, g, wp, n_pad, kc, L.tensor_view(out, co, OFF), None, L.ACT_NONE, 0.0, 1, 1)
    ck.close('fwd accumulate 1', 'fwd_acc', out[..., OFF:OFF + co], prev.double() + pre, kf)
    ck.untouched('fwd accumulate 1', out, co)
    out = out_buf(n, oext, co)
    out[..., OFF:OFF + co] = prev
    L.conv_igemm(xv, g, wp, n_pad, kc, L.tensor_view(out, co, OFF), bias, L.ACT_TANH, 0.0, 1, 2)
    ck.close('fwd accumulate 2 + bias + tanh', 'fwd_sigmoid_tanh', out[..., OFF:OFF + co], torch.tanh(prev.double() + pre + b64), kf,
             fast_math=True)
    ck.untouched('fwd accumulate 2', out, co)
    out = out_buf(n, oext, co)
    out[..., OFF:OFF + co] = 0.0
    L.conv_igemm(xv, g, wp, n_pad, kc, L.tensor_view(out, co, OFF), bias, L.ACT_NONE, 0.0, 3)
    ck.close('fwd split_k 3', 'fwd_split', out[..., OFF:OFF + co], pre + b64, kf)
    ck.untouched('fwd split_k 3', out, co)

    # ---- input gradient: the transposed geometry with the DGRAD-layout pack
    dy = act_input(n, oext, (co + 3) // 4 * 4, None, seed=5)
    dy[..., co:] = NAN
    dyq = tf32(dy, mode)[..., :co].double()
    dyv = L.tensor_view(dy, co)
    dref = ref_conv(dyq, wd, ke, s, p, not transposed, ext)
    dx = out_buf(n, ext, ci_int)
    L.conv_igemm(dyv, gt, wpd, n_pad_d, kc_d, L.tensor_view(dx, ci_int, OFF))
    ck.close('dgrad', 'dgrad', dx[..., OFF:OFF + ci_int], dref, kd)
    ck.untouched('dgrad', dx, ci_int)
    addend, prev_dx = rnd(n, *ext, ci_int, seed=6), rnd(n, *ext, ci_int, seed=7)
    for aux in range(5):
        y = act_output(aux, (n,) + tuple(ext) + (ci_int,), seed=8 + aux)
        der = act_deriv(y, aux)
        for add in (None, addend):
            for acc in (0, 2):
                o = torch.full_like(addend, NAN) if acc == 0 else prev_dx.clone()
                L.conv_igemm_actgrad(dyv, gt, wpd, n_pad_d, kc_d, L.tensor_view(o, ci_int), y.data_ptr(),
                                     0 if add is None else add.data_ptr(), aux, ALPHA, acc)
                v = dref + (0.0 if add is None else add.double()) + (prev_dx.double() if acc == 2 else 0.0)
                ck.close('actgrad aux %d addend %d accumulate %d' % (aux, add is not None, acc), 'actgrad', o, v * der, kd)

    # ---- weight gradient, FWD layout; accumulates into a prefilled buffer, padding rows / columns receive nothing
    wref = ref_wgrad(tf32(x, mode)[..., :ci_int].double(), dyq, ke, s, p, transposed).transpose(1, 2)    # [taps][co][ci]
    full = torch.zeros(taps, n_pad, kc * 32, device='cuda', dtype=torch.float64)
    full[:, :co, :ci_int] = wref
    base = rnd(taps * n_pad * kc * 32, seed=9)
    for split in (0, 1, 2, 3, 7):
        dwp = base.clone()
        L.conv_wgrad(xv, dyv, g, dwp, n_pad, kc, split)
        ck.close('wgrad split_k %d' % split, 'wgrad', (dwp - base).view(taps, n_pad, kc * 32), full, kw)
    ck.done()


@gpu
@pytest.mark.parametrize('case', [MODEL_CASES[1], MODEL_CASES[19], EDGE_CASES[0]], ids=case_id)
def test_exact_mode_matches_fp64_on_raw_operands(L, case):
    """The fp32-exact 3xTF32 mode (conv3x: forward, dgrad, fused activation-gradient dgrad; the three-pass weight gradient)
    against fp64 on the raw fp32 activations and weights: only the dropped lo x lo term (2^-22) and fp32 accumulation remain."""
    from video_prediction_b200.models.savp_model import conv3x
    kind, k, s, p, transposed, ci_ref, ci_int, cmap, co, ext = case
    assert kind == PLAIN and cmap is None and ci_ref == ci_int
    taps = k[0] * k[1] * k[2]
    oext = out_extent(case)
    n = batch_of(ext)
    ck = Checks(case_id(case) + ' [exact]')
    sp = s[0] * s[1] * s[2]
    kf = taps * ci_int / (sp if transposed else 1)          # products per output: forward
    kd = taps * co / (1 if transposed else sp)              # dgrad (the flipped geometry)
    kw = n * (ext[0] * ext[1] * ext[2] if transposed else oext[0] * oext[1] * oext[2])    # wgrad, unsplit
    w = rnd(*k, ci_ref, co, seed=1, scale=(taps * ci_ref) ** -0.5)
    bias = rnd(co, seed=2, scale=0.3)
    w64 = w.double().reshape(taps, ci_ref, co)
    packs = {}
    for layout in (L.WLAYOUT_FWD, L.WLAYOUT_FWD | L.WLAYOUT_RESIDUAL, L.WLAYOUT_DGRAD, L.WLAYOUT_DGRAD | L.WLAYOUT_RESIDUAL):
        packs[layout] = L.pack_weights(w, k, ci_ref, co, kind, layout, ci_int=ci_int)
    (wp, n_pad, kc), (wp_lo, _, _) = packs[L.WLAYOUT_FWD], packs[L.WLAYOUT_FWD | L.WLAYOUT_RESIDUAL]
    (wpd, n_pad_d, kc_d), (wpd_lo, _, _) = packs[L.WLAYOUT_DGRAD], packs[L.WLAYOUT_DGRAD | L.WLAYOUT_RESIDUAL]
    g, gt = L.geom(k, s, p, transposed), L.geom(k, s, p, not transposed)
    x = act_input(n, ext, ci_int, None, seed=3)
    pre = ref_conv(x[..., :ci_int].double(), w64, k, s, p, transposed, oext)
    out = out_buf(n, oext, co)
    conv3x(x, ci_int, g, wp, wp_lo, n_pad, kc, L.tensor_view(out, co, OFF), bias, L.ACT_LRELU, ALPHA)
    ck.close('conv3x forward + bias + lrelu', 'fwd', out[..., OFF:OFF + co], act_ref(pre + bias.double(), L.ACT_LRELU),
             kf, exact=True)
    ck.untouched('conv3x forward', out, co)
    dy = act_input(n, oext, co, None, seed=5)
    dref = ref_conv(dy[..., :co].double(), w64.transpose(1, 2), k, s, p, not transposed, ext)
    dx = out_buf(n, ext, ci_int)
    conv3x(dy, co, gt, wpd, wpd_lo, n_pad_d, kc_d, L.tensor_view(dx, ci_int, OFF), None, L.ACT_NONE, 0.0)
    ck.close('conv3x dgrad', 'dgrad', dx[..., OFF:OFF + ci_int], dref, kd, exact=True)
    y, add = act_output(L.ACT_LRELU, (n,) + tuple(ext) + (ci_int,), seed=8), rnd(n, *ext, ci_int, seed=6)
    o = torch.full_like(add, NAN)
    conv3x(dy, co, gt, wpd, wpd_lo, n_pad_d, kc_d, L.tensor_view(o, ci_int), None, L.ACT_NONE, ALPHA,
           aux=(y.data_ptr(), add.data_ptr(), L.ACT_LRELU))
    ck.close('conv3x actgrad lrelu + addend', 'actgrad', o, (dref + add.double()) * act_deriv(y, L.ACT_LRELU), kd, exact=True)
    # three-pass weight gradient, as ConvLayer.wgrad / SNLayer.wgrad run it: x dy + x_lo dy + x dy_lo
    dwp = torch.zeros(taps * n_pad * kc * 32, device='cuda')
    xv, dyv = L.tensor_view(x, ci_int), L.tensor_view(dy, co)
    L.conv_wgrad(xv, dyv, g, dwp, n_pad, kc, 0)
    L.conv_wgrad(L.tensor_view(L.tf32_residual(x), ci_int), dyv, g, dwp, n_pad, kc, 0)
    L.conv_wgrad(xv, L.tensor_view(L.tf32_residual(dy), co), g, dwp, n_pad, kc, 0)
    wref = ref_wgrad(x[..., :ci_int].double(), dy[..., :co].double(), k, s, p, transposed).transpose(1, 2)
    ck.close('three-pass wgrad', 'wgrad', dwp.view(taps, n_pad, kc * 32)[:, :co, :ci_int], wref, kw, exact=True)
    ck.done()


# ------------------------------------------------------------------ GPU: weight packing
PACK_CASES = sorted({(c[0], c[1], c[5], c[6], c[7], c[8]) for c in MODEL_CASES + EDGE_CASES}, key=str)


def _tf32_ulps(a, b):
    """elementwise distance of two fp32 tensors of equal signs in TF32 ulps (2^13 units of the fp32 bit pattern)"""
    return (a.view(torch.int32).long() - b.view(torch.int32).long()).abs() / 0x2000


@gpu
@pytest.mark.parametrize('pcase', PACK_CASES, ids=lambda c: '%s_k%s_%d-%d_co%d' % ('PMU'[c[0]], ''.join(map(str, c[1])), c[2], c[3], c[5]))
def test_weight_packing(L, pcase):
    """PLAIN: the FWD pack is tf32_rna(w / sigma) permuted by cmap, zero elsewhere -- bit-exact without sigma; with sigma at
    most one TF32 ulp, because the pack kernel divides with the fast (approximate) division of --use_fast_math.
    POOLED / UPSAMPLED: with weights whose effective kernels are exact in TF32 (multiples of 1/16 up to 7/16), the unpacked
    taps convolved by ref_conv reproduce O.conv_pool2d / O.upsample_conv2d in fp64.  DGRAD is the transpose of FWD, bit for
    bit, zero elsewhere; the RESIDUAL pack is tf32_rna(w - tf32_rna(w))."""
    from oracle import savp_oracle as O
    kind, k, ci_ref, ci_int, cmap, co = pcase
    ke = eff_kernel(kind, k)
    taps = ke[0] * ke[1] * ke[2]
    cm = None if cmap is None else torch.tensor(cmap, dtype=torch.int32, device='cuda')
    cmap_l = list(range(ci_int)) if cmap is None else list(cmap)
    src = [i for i, v in enumerate(cmap_l) if v >= 0]
    ref_ch = [cmap_l[i] for i in src]
    if kind == PLAIN:
        w = rnd(*k, ci_ref, co, seed=11)
        for sigma in (None, torch.tensor([1.7], device='cuda')):
            v = w if sigma is None else w / sigma
            eff = torch.zeros(taps, ci_int, co, device='cuda')
            eff[:, src, :] = v.reshape(taps, ci_ref, co)[:, ref_ch, :]
            want = torch.zeros(taps, n_pad_of(L, co), (ci_int + 31) // 32 * 32, device='cuda')
            want[:, :co, :ci_int] = tf32(eff, 'rna').transpose(1, 2)
            wp, n_pad, kc = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_FWD, ci_int=ci_int, cmap=cm, inv_scale=sigma)
            got = wp.view(taps, n_pad, kc * 32)
            if sigma is None:
                assert torch.equal(got, want), 'PLAIN pack differs from tf32_rna(w)[cmap]'
                lo, _, _ = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_FWD | L.WLAYOUT_RESIDUAL, ci_int=ci_int, cmap=cm)
                want_lo = torch.zeros_like(want)
                want_lo[:, :co, :ci_int] = tf32(eff - tf32(eff, 'rna'), 'rna').transpose(1, 2)
                assert torch.equal(lo.view(taps, n_pad, kc * 32), want_lo), 'RESIDUAL pack differs from tf32_rna(w - tf32_rna(w))'
            else:
                ulps = _tf32_ulps(got, want).max().item()
                assert ulps <= 1, 'PLAIN pack with sigma: %d TF32 ulps from tf32_rna(w / sigma)' % ulps
            wpd, n_pad_d, kc_d = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_DGRAD, ci_int=ci_int, cmap=cm, inv_scale=sigma)
            _check_dgrad_pack(got, wpd.view(taps, n_pad_d, kc_d * 32), co, ci_int)
        return
    g = torch.Generator().manual_seed(12)
    w = (torch.randint(-7, 8, (k[1], k[2], ci_ref, co), generator=g).float() / 16).cuda()
    wp, n_pad, kc = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_FWD, ci_int=ci_int, cmap=cm)
    taps_m = unpack(wp, taps, n_pad, kc, co, ci_int)
    x_ref = rnd(2, 9, 11, ci_ref, seed=13).double()
    x_int = torch.zeros(2, 1, 9, 11, ci_int, device='cuda', dtype=torch.float64)
    x_int[..., src] = x_ref[:, None][..., ref_ch]
    zero = torch.zeros(co, device='cuda', dtype=torch.float64)
    if kind == POOLED:
        want = O.conv_pool2d(x_ref, w.double(), zero)
        got = ref_conv(x_int, taps_m, ke, S2, (0, (k[1] - 1) // 2, (k[2] - 1) // 2), False, (1,) + tuple(want.shape[1:3]))
    else:
        want = O.upsample_conv2d(x_ref, w.double(), zero)
        got = ref_conv(x_int, taps_m, ke, S2, (0, 2, 2), True, (1,) + tuple(want.shape[1:3]))
    err = ((got[:, 0] - want).norm() / want.norm()).item()
    WORST['PACK_TOL'] = max(WORST.get('PACK_TOL', (0.0,)), (err, str(pcase)))
    assert err <= PACK_TOL, '%s pack: relative L2 %.3e' % ('POOLED' if kind == POOLED else 'UPSAMPLED', err)
    wpd, n_pad_d, kc_d = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_DGRAD, ci_int=ci_int, cmap=cm)
    _check_dgrad_pack(wp.view(taps, n_pad, kc * 32), wpd.view(taps, n_pad_d, kc_d * 32), co, ci_int)
    lo, _, _ = L.pack_weights(w, k, ci_ref, co, kind, L.WLAYOUT_FWD | L.WLAYOUT_RESIDUAL, ci_int=ci_int, cmap=cm)
    assert float(lo.abs().max()) == 0.0, 'RESIDUAL of TF32-exact weights must be zero'


def n_pad_of(L, rows):
    return L.choose_n_pad(rows)


def _check_dgrad_pack(fwd, dgr, co, ci_int):
    assert torch.equal(dgr[:, :ci_int, :co], fwd[:, :co, :ci_int].transpose(1, 2)), 'DGRAD pack is not the transpose of FWD'
    assert float(dgr[:, ci_int:, :].abs().sum()) == 0.0 and float(dgr[:, :, co:].abs().sum()) == 0.0, 'DGRAD padding not zero'


@gpu
def test_tf32_residual_is_x_minus_truncated_x(L):
    x = torch.cat([rnd(4096, seed=14), rnd(4096, seed=15, scale=1e-30), rnd(4096, seed=16, scale=1e30)])
    assert torch.equal(L.tf32_residual(x), x - tf32(x, 'trunc'))


# ------------------------------------------------------------------ GPU: rejected calls
@gpu
def test_invalid_engine_calls_raise(L):
    x = torch.zeros(1, 8, 8, 40, device='cuda')
    w = rnd(1, 3, 3, 32, 16, seed=1)
    wp, n_pad, kc = L.pack_weights(w, (1, 3, 3), 32, 16, PLAIN, L.WLAYOUT_FWD)
    g = L.geom((1, 3, 3), (1, 1, 1), (0, 1, 1))
    xv = L.tensor_view(x, 32)
    out = torch.zeros(1, 8, 8, 24, device='cuda')
    ov = L.tensor_view(out, 16)
    with pytest.raises(L.VpError, match='split_k needs act NONE'):
        L.conv_igemm(xv, g, wp, n_pad, kc, ov, None, L.ACT_RELU, 0.0, 2)
    with pytest.raises(L.VpError, match='accumulate = 2 needs split_k <= 1'):
        L.conv_igemm(xv, g, wp, n_pad, kc, ov, None, L.ACT_NONE, 0.0, 2, 2)
    with pytest.raises(L.VpError, match='accumulate must be 0, 1 or 2'):
        L.conv_igemm(xv, g, wp, n_pad, kc, ov, None, L.ACT_NONE, 0.0, 1, 3)
    y = torch.zeros_like(out)
    with pytest.raises(L.VpError, match='dense output required'):
        L.conv_igemm_actgrad(xv, g, wp, n_pad, kc, ov, y.data_ptr(), 0, L.ACT_LRELU, 0.2)
    with pytest.raises(L.VpError, match='16B aligned'):
        L.conv_igemm(xv, g, wp, n_pad, kc, L.tensor_view(out, 16, 2))
    torch.cuda.synchronize()
    assert float(out.abs().max()) == 0.0, 'a rejected call wrote its output'


# ------------------------------------------------------------------ GPU: the table covers the model
def _norm_cmap(cm):
    if cm is None:
        return None
    lst = cm.tolist()
    return None if lst == list(range(len(lst))) else tuple(lst)


@gpu
@pytest.mark.parametrize('transformation', ['cdna', 'flow'])
def test_cases_cover_every_model_convolution(L, transformation):
    """Builds the benchmarked configuration (and its flow variant) and requires a MODEL_CASES entry for every generator /
    posterior convolution and every discriminator layer: a new layer geometry fails here until it has a case."""
    if GOLD not in sys.path:
        sys.path.insert(0, GOLD)
    import make_golden_b16 as G
    from oracle import savp_oracle as O
    from video_prediction_b200.models import get_model_class
    hk = dict(G.HK, transformation=transformation)
    hp = O.make_hparams(**hk)
    params, _ = O.init_params(hp, G.SHAPE, seed=0)
    inputs, _ = O.make_synthetic_inputs(hp, 1, G.SHAPE)
    model = get_model_class('savp')(mode='train', hparams_dict=hk)
    model.set_params(params)
    model.build_graph({'images': inputs['images'].permute(1, 0, 2, 3, 4)})
    Bf, ext = model.Bf, {}
    for li, d in enumerate(model.gl):
        ext[id(d['conv'])] = (1,) + tuple(Bf['in%d' % li].shape[2:4])
        if 'rconv' in d:
            ext[id(d['rconv'])] = (1,) + tuple(Bf['rin%d' % li].shape[2:4])
    for c in (model.conv_scratch, model.conv_hmasks, model.conv_simg, model.conv_masks) + \
            ((model.conv_hflow, model.conv_flows) if model.flow else ()):
        ext[id(c)] = (1, model.H, model.W)
    for i, e in enumerate(getattr(model, 'enc_layers', [])):
        ext[id(e['conv'])] = (1,) + tuple((Bf['pairs'] if i == 0 else Bf['epre%d' % (i - 1)]).shape[1:3])
    found = []
    for c in model.convs:
        assert id(c) in ext, 'no input extent known for %s' % c.wname
        found.append(((c.kind, tuple(c.k), tuple(c.stride), tuple(c.pad), bool(c.transposed), c.ci_ref, c.ci_int,
                       _norm_cmap(c.cmap), c.co, ext[id(c)]), c.wname))
    assert model.dnets
    for net in model.dnets.values():
        for li, lay in enumerate(net['layers']):
            e = tuple((net['clip'] if li == 0 else net['feat'][li - 1]).shape[1:4])
            gm = lay.geom
            found.append(((PLAIN, tuple(lay.k3), tuple(lay.stride), (gm.pd, gm.ph, gm.pw), False, lay.cin_ref, lay.cin_int,
                           _norm_cmap(lay.cmap), lay.co, e), lay.wname))
    table = set(MODEL_CASES)
    missing = ['%s: %s' % (name, t) for t, name in found if t not in table]
    assert not missing, 'layer geometries without a case in MODEL_CASES: %s' % missing
