"""CPU tests of the robot-state path (savp_model.py:411-421, 655-658): the state reference (tests/savp_state_oracle.py)
against numpy loops and invariants of the reference, the model's parameter specs, and the synthetic dataset's states."""
import numpy as np
import pytest
import torch

import savp_state_oracle as S
from oracle import savp_oracle as O

SC = 'generator/rnn/savp_cell'
HK_SMALL = dict(context_frames=2, sequence_length=5, nz=4, ngf=8, nef=8)
CFG2 = dict(lr=0.0002, beta1=0.5, beta2=0.999, l1_weight=100.0, l2_weight=0.0, kl_weight=1.0, video_sn_vae_gan_weight=0.1,
            video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, gan_feature_cdist_weight=0.0, state_weight=0.0,
            context_frames=2, sequence_length=12)


def _zero_rnn_states(hp, B, H, W, dt):
    """The zero conv-LSTM states generator_given_z starts from (zero_state, savp_model.py:344-352)."""
    enc, dec = O.layer_specs(hp, H, W)
    out, hh, ww = [], H, W
    for oc, use in enc:
        hh, ww = hh // 2, ww // 2
        if use:
            out.append((torch.zeros(B, hh, ww, oc, dtype=dt), torch.zeros(B, hh, ww, oc, dtype=dt)))
    for oc, use in dec:
        hh, ww = hh * 2, ww * 2
        if use:
            out.append((torch.zeros(B, hh, ww, oc, dtype=dt), torch.zeros(B, hh, ww, oc, dtype=dt)))
    return out, len(enc) + len(dec) + sum(u for _, u in enc + dec)


def test_cell_step_with_actions_and_states_matches_a_numpy_loop(monkeypatch):
    """One cell step in fp64: the select (:411-412), the dense layer state_pred (:655-658), and the vector
    [actions | state | rnn_z] at every tile-concat site (:414-421, :455-469 and the decoder), restated with numpy loops."""
    hp = O.make_hparams(**HK_SMALL)
    A, Sd, B, H, W, nz = 4, 3, 3, 32, 32, hp.nz
    params, _ = S.init_params(hp, (H, W, 3), action_dim=A, state_dim=Sd, dtype=torch.float64)
    rng = np.random.default_rng(5)
    params[SC + '/state_pred/dense/bias'] = torch.tensor(rng.standard_normal(Sd))       # a nonzero bias is checked too
    images = torch.tensor(rng.uniform(size=(B, H, W, 3)))
    action, state_gt, gen_prev = (rng.standard_normal((B, n)) for n in (A, Sd, Sd))
    zs = rng.standard_normal((B, nz))
    gt = np.array([True, False, True])
    conv_states, n_sites = _zero_rnn_states(hp, B, H, W, torch.float64)
    rnn = dict(gen_image=torch.zeros(B, H, W, 3, dtype=torch.float64), conv_rnn_states=conv_states,
               rnn_z_state=(torch.zeros(B, nz, dtype=torch.float64), torch.zeros(B, nz, dtype=torch.float64)),
               gen_state=torch.tensor(gen_prev))
    seen = []
    real = O.tile_concat_z

    def spy(h, z):
        seen.append(z.detach().numpy().copy())
        return real(h, z)
    monkeypatch.setattr(O, 'tile_concat_z', spy)
    inp = dict(images=images, actions=torch.tensor(action), states=torch.tensor(state_gt), zs=torch.tensor(zs))
    with torch.no_grad():
        out, new = S.savp_cell_step(O.Vars(params), hp, SC, 3, inp, images, rnn, torch.tensor(gt))
    # numpy: select, dense LSTM on z from the zero state (savp_model.py:354-362), dense state_pred
    state = np.where(gt[:, None], state_gt, gen_prev)
    K, b = params[SC + '/lstm_z/basic_lstm_cell/kernel'].numpy(), params[SC + '/lstm_z/basic_lstm_cell/bias'].numpy()
    gates = np.concatenate([zs, np.zeros((B, nz))], axis=1) @ K + b
    i, j, f, o = np.split(gates, 4, axis=1)
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))                                       # noqa: E731
    rnn_z = np.tanh(sig(i) * np.tanh(j)) * sig(o)
    Kp, bp = params[SC + '/state_pred/dense/kernel'].numpy(), params[SC + '/state_pred/dense/bias'].numpy()
    x = np.concatenate([action, state], axis=1)
    want = np.zeros((B, Sd))
    for n in range(B):
        for c in range(Sd):
            want[n, c] = bp[c] + sum(x[n, k] * Kp[k, c] for k in range(A + Sd))
    assert np.abs(out['gen_states'].numpy() - want).max() < 1e-12
    assert torch.equal(new['gen_state'], out['gen_states'])
    saz = np.concatenate([action, state, rnn_z], axis=1)
    assert len(seen) == n_sites == 7                                   # 32x32: 4 convolutions, 3 conv-LSTMs
    for z in seen:
        assert z.shape == (B, A + Sd + nz) and np.abs(z - saz).max() < 1e-12


def _with_zero_state_rows(hp, plain, Sd, seed=4):
    """The no-states variables widened to a states model: Sd zero rows after the action rows of every tile-concat kernel,
    and a random state_pred layer."""
    nz = hp.nz
    out = dict(plain)
    shapes, _ = S.init_params(hp, (32, 32, 3), action_dim=4, state_dim=Sd, dtype=torch.float64)
    for k, v in shapes.items():
        if k.startswith(SC + '/state_pred/'):
            out[k] = torch.tensor(np.random.default_rng(seed).standard_normal(tuple(v.shape)))
        elif tuple(v.shape) != tuple(plain[k].shape):
            old = plain[k]
            assert v.shape[2] == old.shape[2] + Sd and v.shape[:2] == old.shape[:2] and v.shape[3:] == old.shape[3:], k
            cut = old.shape[2] - nz - (old.shape[3] // 4 if 'conv2dlstm' in k else 0)    # conv-LSTM rows: [x | z | h]
            zeros = torch.zeros(old.shape[:2] + (Sd,) + old.shape[3:], dtype=old.dtype)
            out[k] = torch.cat([old[:, :, :cut], zeros, old[:, :, cut:]], dim=2)
    return out


@pytest.mark.parametrize('nz', [0, 4])
def test_zero_state_rows_leave_the_images_unchanged(nz):
    """With zero state rows in every tile-concat kernel, the states reference's images are the oracle's without states."""
    hp = O.make_hparams(**dict(HK_SMALL, nz=nz))
    plain, _ = O.init_params(hp, (32, 32, 3), action_dim=4, seed=1, dtype=torch.float64)
    params = _with_zero_state_rows(hp, plain, 3)
    inputs, noise = S.make_synthetic_inputs(hp, 2, (32, 32, 3), action_dim=4, state_dim=3, dtype=torch.float64)
    gt = O.ground_truth_mask(hp, 2)
    with torch.no_grad():
        ref = O.generator(O.Vars(plain), hp, {k: v for k, v in inputs.items() if k != 'states'}, noise, gt)
        out = S.generator(O.Vars(params), hp, inputs, noise, gt)
    keys = ['gen_images'] + (['gen_images_enc'] if nz else [])
    for k in keys:
        assert (out[k] - ref[k]).abs().max().item() < 1e-12, k
    assert set(out) - set(ref) == ({'gen_states', 'gen_states_enc'} if nz else {'gen_states'})
    assert out['gen_states'].shape == (hp.sequence_length - 1, 2, 3)


def test_losses_give_state_pred_and_the_states_no_gradient():
    """stop_gradient on the tile-concat (:414-421) and no loss on gen_states: neither state_pred nor the states input gets a
    gradient, while the generated states feed back over every future step (test-mode mask)."""
    hk = dict(HK_SMALL, l1_weight=1.0, l2_weight=0.5, kl_weight=1.0)
    hp = O.make_hparams(**hk)
    params, _ = S.init_params(hp, (32, 32, 3), action_dim=4, state_dim=3, dtype=torch.float64)
    inputs, noise = S.make_synthetic_inputs(hp, 2, (32, 32, 3), action_dim=4, state_dim=3, dtype=torch.float64)
    P = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    states = inputs['states'].clone().requires_grad_(True)
    inputs['states'] = states
    out = S.generator(O.Vars(P), hp, inputs, noise, O.ground_truth_mask(hp, 2))
    loss = O.total_loss(O.generator_losses(hp, inputs, out, step=3))
    names = [SC + '/state_pred/dense/kernel', SC + '/state_pred/dense/bias']
    grads = torch.autograd.grad(loss, [P[n] for n in names] + [states, P[SC + '/h0/conv_pool2d/kernel']], allow_unused=True)
    assert all(g is None for g in grads[:3]), [g is None for g in grads[:3]]
    assert grads[3] is not None and grads[3].abs().max() > 0
    # the states reach the images: change them and gen_images move
    with torch.no_grad():
        moved = S.generator(O.Vars(params), hp, dict(inputs, states=inputs['states'] + 1.0), noise, O.ground_truth_mask(hp, 2))
    assert (moved['gen_images'] - out['gen_images'].detach()).abs().max() > 0


def test_oracle_train_step_leaves_state_pred_unchanged():
    hk = dict(HK_SMALL, l1_weight=1.0, kl_weight=1.0)
    hp = O.make_hparams(**hk)
    params, _ = S.init_params(hp, (32, 32, 3), action_dim=4, state_dim=3, dtype=torch.float64)
    inputs, noise = S.make_synthetic_inputs(hp, 2, (32, 32, 3), action_dim=4, state_dim=3, dtype=torch.float64)
    opt = dict(m={k: torch.zeros_like(v) for k, v in params.items()}, v={k: torch.zeros_like(v) for k, v in params.items()}, t=0)
    res = S.train_step(params, opt, hp, inputs, noise, step=0)
    assert O.generator is not S.generator                                   # the module is restored
    for n in ('kernel', 'bias'):
        k = SC + '/state_pred/dense/' + n
        assert res['g_grads'][k] is None and torch.equal(res['params'][k], params[k])
    assert 'gen_states' in res['outputs'] and 'gen_states_enc' in res['outputs']


def _model_specs(hk, A, Sd, H=64, W=64):
    from video_prediction_b200.models import SAVPVideoPredictionModel
    m = SAVPVideoPredictionModel(mode='train', hparams_dict=hk)
    m.B, m.T, m.H, m.W, m.C, m.A, m.Sd = 1, hk['sequence_length'], H, W, 3, A, Sd
    m.S, m.Zc = m.T - 1, A + Sd + m.hparams.nz
    m.enc_specs, m.dec_specs = m.layer_specs(m.hparams.ngf, H, W)
    return m._generator_param_specs(), m


def test_param_specs_with_states_follow_the_reference_scopes():
    """cfg2 hparams, A = 4, Sd = 3: 7,603,873 generator variables = 7,496,809 without states + 107,040 tile-concat kernel rows
    + 24 for state_pred; names and shapes agree with the states reference's init_params, also for nz = 0."""
    count = lambda specs: sum(int(np.prod(s)) for s, _ in specs.values())      # noqa: E731
    with_states, _ = _model_specs(CFG2, 4, 3)
    without, _ = _model_specs(CFG2, 4, 0)
    assert count(with_states) == 7603873 and count(without) == 7496809
    assert with_states[SC + '/state_pred/dense/kernel'] == ((7, 3), 'kernel')
    assert with_states[SC + '/state_pred/dense/bias'] == ((3,), 'zeros')
    assert with_states[SC + '/h0/conv_pool2d/kernel'][0] == (5, 5, 2 * 3 + 4 + 3 + 8, 32)
    assert with_states['generator/encoder/layer_1/conv2d/kernel'][0] == (4, 4, 2 * 3 + 4, 64)      # actions only (:21-51)
    for nz in (8, 0):
        hk = dict(CFG2, nz=nz)
        specs, _ = _model_specs(hk, 4, 3)
        ref, _ = S.init_params(O.make_hparams(**{k: v for k, v in hk.items()}), (64, 64, 3), action_dim=4, state_dim=3)
        gen_ref = {k: v for k, v in ref.items() if k.startswith('generator/')}
        assert set(specs) == set(gen_ref), sorted(set(specs) ^ set(gen_ref))[:5]
        for k, (shape, _) in specs.items():
            assert tuple(shape) == tuple(gen_ref[k].shape), k


def test_states_without_actions_and_the_oracle_defaults_are_unchanged():
    hp = O.make_hparams(**HK_SMALL)
    a, _ = O.init_params(hp, (32, 32, 3), seed=2)
    b, _ = S.init_params(hp, (32, 32, 3), seed=2)
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    ia, na = O.make_synthetic_inputs(hp, 2, (32, 32, 3), action_dim=4)
    ib, nb = S.make_synthetic_inputs(hp, 2, (32, 32, 3), action_dim=4, state_dim=2)
    assert set(ib) - set(ia) == {'states'} and all(torch.equal(ia[k], ib[k]) for k in ia)
    assert ib['states'].shape == (hp.sequence_length, 2, 2)
    params, _ = S.init_params(hp, (32, 32, 3), state_dim=2, dtype=torch.float64)
    assert tuple(params[SC + '/state_pred/dense/kernel'].shape) == (2, 2)
    with torch.no_grad():
        out = S.generator(O.Vars(params), hp, {'images': ib['images'].double(), 'states': ib['states'].double()},
                          {k: v.double() for k, v in nb.items() if torch.is_tensor(v)}, O.ground_truth_mask(hp, 2))
    assert out['gen_states'].shape == (hp.sequence_length - 1, 2, 2)


def test_synthetic_dataset_yields_states_with_use_state():
    from video_prediction_b200 import datasets
    DS = datasets.get_dataset_class('synthetic')
    base = DS('none', mode='train', seed=3, hparams='sequence_length=6,action_dim=4').make_batch(2)
    assert set(base) == {'images', 'actions'}
    st = DS('none', mode='train', seed=3, hparams='sequence_length=6,action_dim=4,use_state=True').make_batch(2)
    assert st['states'].shape == (2, 6, 3) and st['states'].dtype == np.float32
    assert all(np.array_equal(base[k], st[k]) for k in base)               # the default draws are unchanged
    st5 = DS('none', mode='train', seed=3, hparams='sequence_length=6,use_state=True,state_dim=5').make_batch(2)
    assert st5['states'].shape == (2, 6, 5) and set(st5) == {'images', 'states'}


def test_model_validates_states_shape():
    from video_prediction_b200.models import SAVPVideoPredictionModel
    imgs = np.zeros((2, 6, 32, 32, 3), np.float32)
    assert SAVPVideoPredictionModel._states_dim({'images': imgs}) == 0
    assert SAVPVideoPredictionModel._states_dim({'images': imgs, 'states': np.zeros((2, 6, 3))}) == 3
    for bad in (np.zeros((2, 5, 3)), np.zeros((1, 6, 3)), np.zeros((2, 6, 0)), np.zeros((2, 6))):
        with pytest.raises(ValueError):
            SAVPVideoPredictionModel._states_dim({'images': imgs, 'states': bad})
