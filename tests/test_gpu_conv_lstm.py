"""GPU tests (-m gpu) of the norm-free ConvLSTM (conv_rnn_norm_layer='none' and ablation_conv_rnn_norm): the gate-interleaved
pack, vp_conv_lstm_fwd against fp64 at every ConvLSTM geometry of the 64x64 and 128x128 models, vp_lstm_plain_bwd against
fp64 autograd, the generator and the training step against the fp32 reference (tests/savp_conv_lstm_oracle.py), and the
captured step."""
import numpy as np
import pytest
import torch

import savp_conv_lstm_oracle as R
import test_gpu_engine as E
from oracle import savp_oracle as O
from test_gpu_engine import L, mode  # noqa: F401  (fixtures of the engine check)
from test_gpu_engine import PLAIN, S1, _case, _norm_cmap
from test_gpu_states import _batch_major
from test_gpu_train_parity import EXACT_GTOL, MODES, _rel, arithmetic, tf32_mode

pytestmark = pytest.mark.gpu
SC = 'generator/rnn/savp_cell'
NAN = float('nan')
VARIANTS = {'none': dict(conv_rnn_norm_layer='none'), 'ablation': dict(ablation_conv_rnn_norm=True)}


@pytest.fixture(scope='module')
def Model(L):  # noqa: F811
    from video_prediction_b200.models import get_model_class
    return get_model_class('savp')


def _gates_perm(F):
    """GEMM column n of a GATES pack -> natural output channel: n = 128 t + 32 g + c holds gate g of cell channel 32 t + c."""
    n = torch.arange(4 * F)
    return ((n % 128) // 32) * F + 32 * (n // 128) + n % 32


# ------------------------------------------------------------------------------------------------ packing
@pytest.mark.parametrize('F', [32, 64, 128, 256])
def test_gates_pack_is_the_permuted_natural_pack(L, F):  # noqa: F811
    ci = 2 * F + 8
    w = E.rnd(5, 5, ci, 4 * F, seed=F, scale=0.1)
    perm = _gates_perm(F).cuda()
    for extra in (0, L.WLAYOUT_RESIDUAL):
        nat, n_pad, kc = L.pack_weights(w, (1, 5, 5), ci, 4 * F, PLAIN, L.WLAYOUT_FWD | extra)
        gat, n_pad2, kc2 = L.pack_weights(w, (1, 5, 5), ci, 4 * F, PLAIN, L.WLAYOUT_FWD | L.WLAYOUT_GATES | extra)
        assert (n_pad, kc) == (n_pad2, kc2) and n_pad == 4 * F
        nat, gat = nat.view(25, n_pad, kc * 32), gat.view(25, n_pad, kc * 32)
        assert torch.equal(gat, nat[:, perm]), (F, extra)
    with pytest.raises(L.VpError):     # F % 32 != 0
        L.pack_weights(E.rnd(5, 5, 8, 4 * 36), (1, 5, 5), 8, 4 * 36, PLAIN, L.WLAYOUT_FWD | L.WLAYOUT_GATES)
    with pytest.raises(L.VpError):     # not a forward layout
        L.pack_weights(w, (1, 5, 5), ci, 4 * F, PLAIN, L.WLAYOUT_DGRAD | L.WLAYOUT_GATES)


# ------------------------------------------------------------------------------------------------ vp_conv_lstm_fwd
def _lstm_case(hw, F, zc=8):
    return _case(PLAIN, (1, 5, 5), S1, (0, 2, 2), False, 2 * F + zc, 4 * F, (1, hw, hw))


# the gate convolutions of the ConvLSTMs of the 64x64 (ngf 32) and 128x128 generators, nz 8: (x | z | h) -> 4F
LSTM_CASES = sorted(set(_lstm_case(hw, F) for hw, F in ((32, 32), (16, 64), (8, 128),                             # 64x64
                                                      (32, 64), (16, 128), (8, 256), (16, 256), (32, 128))),   # 128x128
                    key=str)


def _cell64(z, c, fb=1.0):
    F = c.shape[-1]
    i, j, f, o = z[..., :F], z[..., F:2 * F], z[..., 2 * F:3 * F], z[..., 3 * F:]
    c2 = c * torch.sigmoid(f + fb) + torch.sigmoid(i) * torch.tanh(j)
    return c2, torch.tanh(c2) * torch.sigmoid(o)


def _run_lstm(L, x, ci, wp, wp_lo, n_pad, kc, bias, c_prev, nb, hw, F, exact):  # noqa: F811
    """One cell step into NaN-prefilled z / c_new and three h destinations (channel slices [4, 4 + F) of F + 8 wide
    NaN buffers).  Returns (z, c_new, [h buffers])."""
    z = torch.full((nb, hw, hw, 4 * F), NAN, device='cuda')
    c_new = torch.full((nb, hw, hw, F), NAN, device='cuda')
    hb = [torch.full((nb, hw, hw, F + 8), NAN, device='cuda') for _ in range(3)]
    dests = [(h.data_ptr() + 16, F + 8) for h in hb]
    x4 = x.view(nb, hw, hw, -1)
    xv, g = L.tensor_view(x4, ci), L.geom((1, 5, 5), (1, 1, 1), (0, 2, 2))
    if exact:
        z.zero_()
        L.conv_lstm_fwd(xv, g, wp, n_pad, kc, z, bias, c_prev, c_new, dests, accumulate=1)
        L.conv_lstm_fwd(L.tensor_view(L.tf32_residual(x4), ci), g, wp, n_pad, kc, z, bias, c_prev, c_new, dests, accumulate=1)
        L.conv_lstm_fwd(xv, g, wp_lo, n_pad, kc, z, bias, c_prev, c_new, dests, accumulate=2)
    else:
        L.conv_lstm_fwd(xv, g, wp, n_pad, kc, z, bias, c_prev, c_new, dests)
    return z, c_new, hb


@pytest.mark.parametrize('nb', [1, 37, 32])
@pytest.mark.parametrize('case', LSTM_CASES, ids=E.case_id)
def test_conv_lstm_fwd_matches_fp64(L, mode, case, nb):  # noqa: F811
    """z against an fp64 convolution of the operands the tensor core reads (the TF32 activations and the packed weights read
    back in natural order) + bias: max-abs <= 5e-6 x max |x| |W| (fp32 accumulation over up to 13,000 products, measured
    worst 2.1e-6 on an H100; a wrong tap or gate would be ~1/25 of that scale).  c_new and h against the fp64 cell evaluated
    on the kernel's own z: <= 2e-5 (fast-math sigmoid / tanh, measured worst 1.0e-5).  The NaN around every h slice stays;
    a rerun gives identical bits."""
    _, k, s, p, _, _, ci, _, co, ext = case
    F, hw = co // 4, ext[1]
    x = E.act_input(nb, ext, ci, None, seed=1)
    w = E.rnd(5, 5, ci, co, seed=2, scale=0.03)
    bias = E.rnd(co, seed=3, scale=0.5)
    c_prev = E.rnd(nb, hw, hw, F, seed=4)
    nat, n_pad, kc = L.pack_weights(w, k, ci, co, PLAIN, L.WLAYOUT_FWD)
    wp, _, _ = L.pack_weights(w, k, ci, co, PLAIN, L.WLAYOUT_FWD | L.WLAYOUT_GATES)
    z, c_new, hb = _run_lstm(L, x, ci, wp, None, n_pad, kc, bias, c_prev, nb, hw, F, False)
    W = E.unpack(nat, 25, n_pad, kc, co, ci)
    xq = E.tf32(x[..., :ci], mode).double()
    ref = E.ref_conv(xq, W, k, s, p, False, ext).view(nb, hw, hw, co) + bias.double()
    scale = E.ref_conv(xq.abs(), W.abs(), k, s, p, False, ext).max()
    c_ref, h_ref = _cell64(z.double(), c_prev.double())
    errs = torch.stack([(z.double() - ref).abs().max() / scale, (c_new.double() - c_ref).abs().max(),
                        max((h[..., 4:4 + F].double() - h_ref).abs().max() for h in hb)]).tolist()
    untouched = all(bool(torch.isnan(h[..., :4]).all() and torch.isnan(h[..., 4 + F:]).all()) for h in hb)
    assert errs[0] <= 5e-6 and errs[1] <= 2e-5 and errs[2] <= 2e-5, errs
    assert untouched
    z2, c2, hb2 = _run_lstm(L, x, ci, wp, None, n_pad, kc, bias, c_prev, nb, hw, F, False)
    assert torch.equal(z, z2) and torch.equal(c_new, c2) and all(torch.equal(a[..., 4:4 + F], b[..., 4:4 + F]) for a, b in zip(hb, hb2))


@pytest.mark.parametrize('case', [LSTM_CASES[0], LSTM_CASES[-1]], ids=E.case_id)
def test_conv_lstm_fwd_exact_mode_matches_fp64_on_raw_operands(L, case):  # noqa: F811
    """The three TF32 passes of the fp32-exact mode (two partial passes, then the residual-weight pass with the cell) against
    fp64 on the raw fp32 operands: z <= 5e-6 x max |x| |W| (measured worst 1.1e-6: the residual passes remove the operand
    rounding, what is left is fp32 accumulation), c_new and h on the kernel's z <= 2e-5 as above."""
    _, k, s, p, _, _, ci, _, co, ext = case
    F, hw, nb = co // 4, ext[1], 37
    x = E.act_input(nb, ext, ci, None, seed=5)
    w = E.rnd(5, 5, ci, co, seed=6, scale=0.03)
    bias = E.rnd(co, seed=7, scale=0.5)
    c_prev = E.rnd(nb, hw, hw, F, seed=8)
    wp, n_pad, kc = L.pack_weights(w, k, ci, co, PLAIN, L.WLAYOUT_FWD | L.WLAYOUT_GATES)
    wp_lo, _, _ = L.pack_weights(w, k, ci, co, PLAIN, L.WLAYOUT_FWD | L.WLAYOUT_GATES | L.WLAYOUT_RESIDUAL)
    z, c_new, hb = _run_lstm(L, x, ci, wp, wp_lo, n_pad, kc, bias, c_prev, nb, hw, F, True)
    W = w.double().view(25, ci, co)
    xr = x[..., :ci].double()
    ref = E.ref_conv(xr, W, k, s, p, False, ext).view(nb, hw, hw, co) + bias.double()
    scale = E.ref_conv(xr.abs(), W.abs(), k, s, p, False, ext).max()
    c_ref, h_ref = _cell64(z.double(), c_prev.double())
    errs = torch.stack([(z.double() - ref).abs().max() / scale, (c_new.double() - c_ref).abs().max(),
                        (hb[0][..., 4:4 + F].double() - h_ref).abs().max()]).tolist()
    assert errs[0] <= 5e-6 and errs[1] <= 2e-5 and errs[2] <= 2e-5, errs


def test_conv_lstm_fwd_rejects_bad_calls(L):  # noqa: F811
    F, hw, nb = 32, 8, 2
    ci = 2 * F + 8
    x = E.rnd(nb, hw, hw, ci)
    w = E.rnd(5, 5, ci, 4 * F, scale=0.03)
    wp, n_pad, kc = L.pack_weights(w, (1, 5, 5), ci, 4 * F, PLAIN, L.WLAYOUT_FWD | L.WLAYOUT_GATES)
    z, c, cn = torch.zeros(nb, hw, hw, 4 * F, device='cuda'), E.rnd(nb, hw, hw, F), torch.zeros(nb, hw, hw, F, device='cuda')
    h = torch.zeros(nb, hw, hw, F, device='cuda')
    bias = torch.zeros(4 * F, device='cuda')
    g = L.geom((1, 5, 5), (1, 1, 1), (0, 2, 2))
    xv = L.tensor_view(x, ci)
    one = [(h.data_ptr(), F)]
    L.conv_lstm_fwd(xv, g, wp, n_pad, kc, z, bias, c, cn, one)                    # the good call
    torch.cuda.synchronize()
    F2 = 36                                                                       # F % 32 != 0
    z2, c2 = torch.zeros(nb, hw, hw, 4 * F2, device='cuda'), torch.zeros(nb, hw, hw, F2, device='cuda')
    bad = [
        lambda: L.conv_lstm_fwd(xv, g, wp, 4 * F2, kc, z2, torch.zeros(4 * F2, device='cuda'), c2, c2.clone(), [(c2.data_ptr(), F2)]),
        lambda: L.conv_lstm_fwd(xv, g, wp, n_pad, kc, z, bias, None, cn, one),   # null c_prev
        lambda: L.conv_lstm_fwd(xv, g, wp, n_pad, kc, z, None, c, cn, one),      # null bias
        lambda: L.conv_lstm_fwd(xv, g, wp, n_pad, kc, z, bias, c, cn, one * 4),  # four destinations
        lambda: L.conv_lstm_fwd(xv, g, wp, n_pad, kc, z, bias, c, cn, []),       # none
        lambda: L.conv_lstm_fwd(xv, g, wp, n_pad, kc, z, bias, c, cn, [(h.data_ptr(), F - 4)]),   # stride below F
        lambda: L.conv_lstm_fwd(xv, g, wp, n_pad, kc, z, bias, c, cn, one, accumulate=3),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(L.VpError):
            call()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ vp_lstm_plain_bwd
@pytest.mark.parametrize('F,rows,nsrc,with_dc', [(32, 37 * 64, 2, True), (128, 2 * 256, 1, False), (256, 37 * 64, 4, True)])
def test_lstm_plain_bwd_matches_fp64_autograd(L, F, rows, nsrc, with_dc):  # noqa: F811
    """dz and dc_prev within 3e-5 of max |ref| (fast-math sigmoid / tanh, measured worst 1.1e-5); reruns are bit-identical."""
    z = E.rnd(rows, 4 * F, seed=1, scale=1.5)
    c_prev = E.rnd(rows, F, seed=2)
    c_new = _cell64(z.double(), c_prev.double())[0].float()
    srcs = [E.rnd(rows, F + 4 * s, seed=10 + s) for s in range(nsrc)]       # channel slices of wider buffers
    dc_next = E.rnd(rows, F, seed=3) if with_dc else None
    z64, c64 = z.double().requires_grad_(True), c_prev.double().requires_grad_(True)
    F_ = F
    i, j, f, o = z64[:, :F_], z64[:, F_:2 * F_], z64[:, 2 * F_:3 * F_], z64[:, 3 * F_:]
    # the kernel reads the stored c_new: differentiate h through it, c_new through the gates
    cn = c64 * torch.sigmoid(f + 1.0) + torch.sigmoid(i) * torch.tanh(j)
    cs = c_new.double().requires_grad_(True)
    h = torch.tanh(cs) * torch.sigmoid(o)
    dh = sum(s[:, :F].double() for s in srcs)
    (dcs, do_) = torch.autograd.grad(h, (cs, z64), dh)
    dc = dcs + (dc_next.double() if with_dc else 0.0)
    dz_ref, dc_ref = torch.autograd.grad(cn, (z64, c64), dc)
    dz_ref = dz_ref + do_
    runs = []
    for _ in range(2):
        dz = torch.full((rows, 4 * F), NAN, device='cuda')
        dcp = torch.full((rows, F), NAN, device='cuda')
        L.lstm_plain_bwd(z, c_prev, c_new, rows, F, [(s.data_ptr(), s.shape[1]) for s in srcs], dc_next, dz, dcp)
        runs.append((dz, dcp))
    for got, ref in ((runs[0][0], dz_ref), (runs[0][1], dc_ref)):
        err = ((got.double() - ref).abs().max() / ref.abs().max()).item()
        assert err <= 3e-5, err
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


# ------------------------------------------------------------------------------------------------ model level
def _params(hp, shape, A=0, seed=0):
    """Reference initial values with a random gate bias (zeros at init) and, for the ablation, a random output norm."""
    params, _ = R.init_params(hp, shape, action_dim=A, seed=seed)
    g = torch.Generator().manual_seed(seed + 11)
    for k in list(params):
        if k.endswith('basic_conv2dlstm_cell/bias'):
            params[k] = torch.randn(params[k].shape, generator=g) * 0.3
        elif '/lstm_h' in k and '/InstanceNorm/' in k:
            params[k] = params[k] + torch.randn(params[k].shape, generator=g) * 0.2
    return params


@pytest.mark.parametrize('variant', sorted(VARIANTS))
def test_lstm_cases_cover_every_convolution(Model, variant):
    """Every convolution of the cfg2 64x64 norm-free model has an engine case: its gate convolutions in LSTM_CASES, all
    others in MODEL_CASES."""
    import make_golden_b16 as G
    hk = dict(G.HK, **VARIANTS[variant])
    hp = O.make_hparams(**hk)
    inputs, _ = O.make_synthetic_inputs(hp, 1, G.SHAPE)
    model = Model(mode='train', hparams_dict=hk)
    model.set_params(R.init_params(hp, G.SHAPE, seed=0)[0])
    model.build_graph(_batch_major(inputs))
    Bf, ext, gates = model.Bf, {}, set()
    for li, d in enumerate(model.gl):
        ext[id(d['conv'])] = (1,) + tuple(Bf['in%d' % li].shape[2:4])
        if 'rconv' in d:
            ext[id(d['rconv'])] = (1,) + tuple(Bf['rin%d' % li].shape[2:4])
            gates.add(id(d['rconv']))
            assert d['rconv'].fwd_layout & L_GATES() and 'gst1_%d' % li not in Bf
    for c in (model.conv_scratch, model.conv_hmasks, model.conv_simg, model.conv_masks):
        ext[id(c)] = (1, model.H, model.W)
    for i, e in enumerate(getattr(model, 'enc_layers', [])):
        ext[id(e['conv'])] = (1,) + tuple((Bf['pairs'] if i == 0 else Bf['epre%d' % (i - 1)]).shape[1:3])
    missing = []
    for c in model.convs:
        t = (c.kind, tuple(c.k), tuple(c.stride), tuple(c.pad), bool(c.transposed), c.ci_ref, c.ci_int, _norm_cmap(c.cmap), c.co,
             ext[id(c)])
        if t not in (set(LSTM_CASES) if id(c) in gates else set(E.MODEL_CASES)):
            missing.append('%s: %s' % (c.wname, t))
    assert len(gates) == 5 and not missing, missing


def L_GATES():
    from video_prediction_b200 import lib
    return lib.WLAYOUT_GATES


GEN_CASES = {
    'deterministic': (dict(context_frames=2, sequence_length=12, nz=0), 4, (64, 64, 3)),
    'vae': (dict(context_frames=2, sequence_length=12, nz=8), 4, (64, 64, 3)),
    'deterministic_128': (dict(context_frames=2, sequence_length=6, nz=0), 2, (128, 128, 3)),
}


@pytest.mark.parametrize('variant', sorted(VARIANTS))
@pytest.mark.parametrize('case', sorted(GEN_CASES))
def test_generator_matches_oracle(Model, case, variant):
    """gen_images (and gen_images_enc) within 1e-3 max-abs of the fp32 reference, as test_gpu_parity.py (measured on an
    H100: 1.5e-4 to 3.1e-4)."""
    hk, B, shape = GEN_CASES[case]
    hk = dict(hk, **VARIANTS[variant])
    hp = O.make_hparams(**hk)
    params = _params(hp, shape)
    inputs, noise = O.make_synthetic_inputs(hp, B, shape, seed=0)
    with torch.no_grad():
        ref = R.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, B, None))
    model = Model(mode='test', hparams_dict=hk)
    model.set_params(params)
    binp = _batch_major(inputs)
    model.build_graph(binp)
    model.set_inputs(binp, noise, sampling=False)
    model.generator_forward()
    torch.cuda.synchronize()
    report = {}
    for k in ('gen_images', 'gen_images_enc') if hp.nz else ('gen_images',):
        err = (model.outputs_time_major(k).cpu() - ref[k]).abs().max().item()
        report[k] = err
        assert err <= 1e-3, (case, variant, k, err)
    print('conv-lstm %s generator %s: max-abs %s' % (variant, case, {k: '%.2e' % v for k, v in report.items()}))


TRAIN_CASES = {
    'vae_l1': dict(context_frames=2, sequence_length=8, nz=8, l1_weight=1.0, kl_weight=1e-3, kl_anneal_steps=(0, 10), lr=1e-3),
    'savp': dict(context_frames=2, sequence_length=8, clip_length=6, lr=2e-4, beta1=0.5, l1_weight=100., kl_weight=1.0,
                 video_sn_vae_gan_weight=0.1, video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, kl_anneal_steps=(0, 10)),
}


def _oracle_step(hp, params, inputs, noise, step, sampling, quant):
    O.set_tf32_emulation(quant)
    try:
        opt = dict(m={k: torch.zeros_like(v) for k, v in params.items()}, v={k: torch.zeros_like(v) for k, v in params.items()}, t=0)
        return R.train_step(params, opt, hp, inputs, noise, step=step, sampling=sampling)
    finally:
        O.set_tf32_emulation(None)


@pytest.mark.parametrize('arith', ['tf32', 'exact'])
@pytest.mark.parametrize('variant', sorted(VARIANTS))
@pytest.mark.parametrize('case', sorted(TRAIN_CASES))
def test_training_step_matches_fp32_oracle(Model, case, variant, arith):
    """64x64, B = 2, random scheduled-sampling mask, the tolerances of test_gpu_train_parity.py: exact mode EXACT_GTOL per
    gradient tensor (2e-3 VAE-L1, 1e-2 with the GANs), TF32 mode max(5e-2, 2 x the operand-rounding emulation).  Measured
    worst relative L2 error on an H100, both variants: exact 7.9e-4 (VAE-L1) and 1.2e-3 (SAVP); TF32 1.5e-2 (VAE-L1) and
    6.1e-2 against a tolerance of 1.1e-1 (SAVP, a discriminator kernel)."""
    hk = dict(TRAIN_CASES[case], **VARIANTS[variant])
    hp = O.make_hparams(**hk)
    B, step, shape = 2, 5, (64, 64, 3)
    params = _params(hp, shape)
    inputs, noise = O.make_synthetic_inputs(hp, B, shape)
    sampling = torch.rand(hp.sequence_length - 1 - hp.context_frames, B, generator=torch.Generator().manual_seed(7)) < 0.5
    _, ltol, floor, otol = MODES[arith]
    with arithmetic(arith):
        model = Model(mode='train', hparams_dict=hk)
        model.set_params(params)
        model.build_graph(_batch_major(inputs))
    model.global_step = step
    model.train_step(_batch_major(inputs), noise, sampling=sampling)
    torch.cuda.synchronize()
    lv = model.losses()
    res = _oracle_step(hp, params, inputs, noise, step, sampling, None)
    emu = _oracle_step(hp, params, inputs, noise, step, sampling, tf32_mode()) if arith == 'tf32' else None
    ref_l = dict(res['g_losses'])
    ref_l.update(res.get('d_losses', {}))
    emu_l = {} if emu is None else dict(emu['g_losses'], **emu.get('d_losses', {}))
    for k, v in ref_l.items():
        tol = max(ltol * abs(v), 2.0 * abs(emu_l[k] - v) if emu_l else 0.0)
        assert abs(lv[k] - v) <= tol + 1e-6, (k, lv[k], v, emu_l.get(k))
    worst, bad = [], []
    for kind in ('g_grads', 'd_grads'):
        if kind not in res:
            continue
        items = [(k, g) for k, g in res[kind].items() if g is not None]
        gmax = max(g.double().norm().item() for _, g in items)
        for k, g in items:
            r, n = _rel(model.grads[k], g)
            if n < floor * gmax:
                continue
            tol = EXACT_GTOL[case] if emu is None else max(5e-2, 2.0 * _rel(emu[kind][k], g)[0])
            worst.append((r, tol, k))
            if r > tol:
                bad.append((r, tol, k))
    worst.sort(reverse=True)
    print('conv-lstm %s %s [%s]: worst gradient errors %s' % (variant, case, arith,
                                                                ['%.2e (tol %.2e) %s' % w for w in worst[:4]]))
    assert not bad, bad[:5]
    lstm = [k for k in res['g_grads'] if k.endswith('basic_conv2dlstm_cell/bias') or ('/lstm_h' in k and '/InstanceNorm/' in k)]
    assert lstm and all(float(model.grads[k].abs().max()) > 0 for k in lstm), lstm     # the new variables are trained
    for k in ('gen_images', 'gen_images_enc'):
        err = (model.outputs_time_major(k).cpu() - res['outputs'][k]).abs().max().item()
        assert err <= otol, (k, err)


@pytest.mark.parametrize('variant', sorted(VARIANTS))
def test_captured_step_reproduces_the_eager_step(Model, variant, tmp_path):
    """The eager step and two graph replays from the same checkpoint give bit-identical losses and gradients."""
    hk = dict(TRAIN_CASES['savp'], **VARIANTS[variant])
    hp = O.make_hparams(**hk)
    params = _params(hp, (64, 64, 3))
    inputs, _ = O.make_synthetic_inputs(hp, 2, (64, 64, 3))
    binp = _batch_major(inputs)
    runs = {}
    for how in ('eager', 'graph'):
        model = Model(mode='train', hparams_dict=hk)
        model.set_params(params)
        model.build_graph(binp)
        model.use_cuda_graph = how == 'graph'
        model.train_step(binp)
        ck = model.save(str(tmp_path / how))
        runs[how] = []
        for _ in range(2 if how == 'graph' else 1):
            model.restore(None, ck)
            model.train_step(binp)
            torch.cuda.synchronize()
            assert (model._graph is not None) == (how == 'graph')
            runs[how].append((model.loss_vals.clone(), model.g_grad.clone(), model.d_grad.clone()))
    ref = runs['eager'][0]
    for got in runs['graph']:
        for name, a, b in zip(('losses', 'g_grad', 'd_grad'), got, ref):
            assert torch.equal(a, b), (name, (a - b).abs().max().item())
    assert float(ref[1].abs().max()) > 0 and bool(torch.isfinite(ref[1]).all())
    np.testing.assert_array_equal(runs['graph'][0][0].cpu().numpy(), runs['graph'][1][0].cpu().numpy())
