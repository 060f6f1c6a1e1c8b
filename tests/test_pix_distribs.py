"""CPU tests of the pixel-distribution path (savp_model.py:408-410, 598-621, 648-653): `pixel_distribution` of the oracle
and of the BAIR reader against a direct loop (tf_utils.py:562-585, quirks included), `object_pos` records parsed under time
shift and frame skip (softmotion_dataset.py:41-42, 59-68), and invariants of the pix-path reference (savp_pix_oracle.py)."""
import os

import numpy as np
import pytest
import torch

import savp_pix_oracle as P
from oracle import savp_oracle as O
from video_prediction_b200 import datasets
from video_prediction_b200.datasets import tfrecord as R
from video_prediction_b200.datasets.video_datasets import pixel_distribution as ds_pixel_distribution


def loop_pixel_distribution(pos, h, w):
    """tf_utils.pixel_distribution restated with scalar loops: four one-hots of flat indices, bilinear weights."""
    out = np.zeros((len(pos), h * w))
    for i, (y, x) in enumerate(pos):
        x0, y0 = int(np.floor(x)), int(np.floor(y))
        for yy, xx, wgt in ((y0, x0, (x0 + 1 - x) * (y0 + 1 - y)), (y0 + 1, x0, (x0 + 1 - x) * (y - y0)),
                            (y0, x0 + 1, (x - x0) * (y0 + 1 - y)), (y0 + 1, x0 + 1, (x - x0) * (y - y0))):
            idx = yy * w + xx
            if 0 <= idx < h * w:
                out[i, idx] += wgt
    return out.reshape(len(pos), h, w)


POS = np.array([[3.0, 5.0],        # integer: a one-hot
                [2.25, 4.5],       # inside: four weights summing to 1
                [1.5, 7.25],       # x1 = W = 8: column 0 of the next row
                [-3.0, 2.0],       # above the frame: nothing
                [9.5, 1.5],        # below the frame: nothing
                [0.0, -0.5],       # x0 = -1 on row 0: flat index -1 drops, x1 = 0 stays
                [6.75, 7.5]])      # last row, last column: the wrapped neighbours run past H*W


@pytest.mark.parametrize('impl', ['oracle', 'dataset'])
def test_pixel_distribution_matches_a_direct_loop(impl):
    h, w = 7, 8
    want = loop_pixel_distribution(POS, h, w)
    if impl == 'oracle':
        got = P.pixel_distribution(torch.tensor(POS, dtype=torch.float64), h, w).numpy()
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-15)
    else:
        got = ds_pixel_distribution(POS, h, w)
        assert got.dtype == np.float32
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-6)
    assert got[0].sum() == 1.0 and got[0, 3, 5] == 1.0                   # integer position: one-hot
    assert abs(got[1].sum() - 1.0) < 1e-6 and got[1, 2:4, 4:6].min() > 0  # inside the frame: weights sum to 1
    assert got[2, 2, 0] > 0 and got[2, 1, 0] == 0                         # x = W wraps into column 0 of the next row
    assert got[3].sum() == 0 and got[4].sum() == 0                        # outside the frame: all zeros
    assert got[5, 0, 0] > 0 and abs(got[5].sum() - 0.5) < 1e-6           # the index -1 contributes nothing
    assert abs(got[6].sum() - 0.125) < 1e-6 and got[6, 6, 7] > 0        # only (6, 7) lies inside: wa = 0.5 * 0.25


def _write_bair_with_object_pos(root, split, ntraj=3, length=30, side=8, ndes=2):
    d = os.path.join(root, split)
    os.makedirs(d)
    recs = []
    for k in range(ntraj):
        f = {}
        for t in range(length):
            f['%d/image_aux1/encoded' % t] = bytes([(k * 40 + t) % 256]) * (side * side * 3)
            f['%d/endeffector_pos' % t] = np.array([k, t, 0.5], np.float32)
            # designated pixel j at (y, x) = (j + 0.5, t / 8): moves right over time, wraps at the row end
            f['%d/object_pos' % t] = np.array([v for j in range(ndes) for v in (j + 0.5, (t % 16) * 0.5)], np.float32)
            if t < length - 1:
                f['%d/action' % t] = np.array([k, t, -t, 1.0], np.float32)
        recs.append(R.make_example(f))
    R.write_records(os.path.join(d, 'traj_0_to_%d.tfrecords' % (ntraj - 1)), recs)


def test_bair_object_pos_yields_pix_distribs_under_time_shift_and_frame_skip(tmp_path):
    root = str(tmp_path / 'bair')
    _write_bair_with_object_pos(root, 'train')
    ds = datasets.SoftmotionVideoDataset(root, mode='train', seed=1, hparams_dict={'use_state': True, 'frame_skip': 1,
                                                                                   'sequence_length': 6})
    assert ds.state_like_names_and_shapes['object_pos'] == ('%d/object_pos', (4,))
    b = ds.make_batch(2)
    assert b['pix_distribs'].shape == (2, 6, 8, 8, 2) and b['pix_distribs'].dtype == np.float32
    for i in range(2):
        frames = b['states'][i, :, 1].astype(int)                          # the source frame of every sampled step
        assert frames[0] % 2 == 0 and (np.diff(frames) == 2).all()          # time shift 2, frame skip 1
        for j in range(2):
            pos = np.array([[j + 0.5, (t % 16) * 0.5] for t in frames])
            np.testing.assert_allclose(b['pix_distribs'][i, ..., j], loop_pixel_distribution(pos, 8, 8), rtol=0, atol=1e-6)
            np.testing.assert_array_equal(b['object_pos'][i, :, 2 * j + 1], pos[:, 1])
    with pytest.raises(NotImplementedError):
        datasets.SoftmotionVideoDataset(root, mode='train', hparams_dict={'crop_size': 6})
    ds2 = datasets.SoftmotionVideoDataset(root, mode='train', hparams_dict={'crop_size': 8})   # no size change: allowed
    assert 'pix_distribs' in ds2.make_batch(1)


def test_bair_without_object_pos_has_no_pix_distribs(tmp_path):
    from test_datasets import _write_bair
    root = str(tmp_path / 'bair')
    _write_bair(root, 'test', ntraj=2)
    b = datasets.SoftmotionVideoDataset(root, mode='test', hparams_dict={'sequence_length': 5}).make_batch(1)
    assert sorted(b) == ['images']


# ------------------------------------------------------------------------------------------------ oracle invariants
def make_pix(hp, B, H, W, D, seed=0, dtype=torch.float64):
    """[T,B,H,W,D] maps of D designated pixels moving along random straight lines, softened with a blurred copy so that no
    plane is a bare one-hot (every plane sums to 1)."""
    rng = np.random.default_rng(seed)
    T = hp.sequence_length
    out = torch.zeros(T, B, H, W, D, dtype=dtype)
    for b in range(B):
        for d in range(D):
            p0 = rng.uniform(0.25, 0.75, 2) * (H - 1, W - 1)
            v = rng.uniform(-1.5, 1.5, 2)
            pos = torch.tensor(np.array([p0 + v * t for t in range(T)]), dtype=dtype)
            m = P.pixel_distribution(pos, H, W)
            blur = torch.nn.functional.avg_pool2d(m[:, None], 3, 1, 1, count_include_pad=False)[:, 0]
            m = 0.5 * m + 0.5 * blur / blur.sum(dim=(1, 2), keepdim=True)
            out[:, b, :, :, d] = m
    return out


def _oracle(hk, B=2, shape=(32, 32, 3), D=2, A=0, pix=None, sampling=None, seed=0):
    hp = O.make_hparams(**hk)
    params, _ = O.init_params(hp, shape, action_dim=A, seed=seed, dtype=torch.float64)
    inputs, noise = O.make_synthetic_inputs(hp, B, shape, action_dim=A, seed=seed, dtype=torch.float64)
    if hk.get('transformation') == 'flow':       # fresh flows are ~0: give them sub-pixel displacements
        params['generator/rnn/savp_cell/flows/conv2d/bias'] = torch.tensor([0.37, 1.27, -0.53, 2.17, 0.61, -1.41, 0.23, 1.79],
                                                                           dtype=torch.float64)
    gt = O.ground_truth_mask(hp, B, sampling)
    with torch.no_grad():
        plain = O.generator(O.Vars(params), hp, inputs, noise, gt)
        inputs['pix_distribs'] = make_pix(hp, B, shape[0], shape[1], D) if pix is None else pix(hp, B, shape)
        out = P.generator(O.Vars(params), hp, inputs, noise, gt)
    return hp, params, inputs, noise, plain, out


HK_SMALL = dict(context_frames=2, sequence_length=5, nz=4, ngf=8, nef=8)


@pytest.mark.parametrize('transformation', ['cdna', 'flow'])
def test_oracle_pix_planes_sum_to_one_and_leave_the_images_alone(transformation):
    hp, _, _, _, plain, out = _oracle(dict(HK_SMALL, transformation=transformation))
    for k in ('gen_pix_distribs', 'gen_pix_distribs_enc'):
        s = out[k].sum(dim=(2, 3))                                         # [T-1, B, D]
        assert (s - 1).abs().max() < 1e-12, (k, s)
        assert out[k].shape == (hp.sequence_length - 1, 2, 32, 32, 2)
    assert out['transformed_pix_distribs'].shape == (hp.sequence_length - 1, 2, 32, 32, 2, 7)
    for k, v in plain.items():                                             # images, masks, zs: untouched by the maps
        assert torch.equal(out[k], v), k
    assert set(out) - set(plain) == {'gen_pix_distribs', 'transformed_pix_distribs', 'gen_pix_distribs_enc',
                                     'transformed_pix_distribs_enc'}


def test_oracle_losses_do_not_depend_on_pix_distribs():
    """No loss reads the maps (base_model.py:733-852): the generator losses of the pix reference's outputs are those of the
    SAVP oracle's."""
    hk = dict(HK_SMALL, l1_weight=1.0, l2_weight=0.5, kl_weight=1.0)
    hp, _, inputs, _, plain, out = _oracle(hk, D=1)
    a, b = O.generator_losses(hp, inputs, plain, step=3), O.generator_losses(hp, inputs, out, step=3)
    assert list(a) == list(b) and list(a)
    for k in a:
        assert torch.equal(a[k][0], b[k][0]) and a[k][1] == b[k][1], k


@pytest.mark.parametrize('transformation', ['cdna', 'flow'])
def test_oracle_constant_plane_stays_constant(transformation):
    """A uniform map is a fixed point: CDNA kernels are normalised, zero flow is the identity, every slot holds the same
    constant and the masks sum to 1."""
    def const(hp, B, shape):
        return torch.full((hp.sequence_length, B, shape[0], shape[1], 1), 1.0 / (shape[0] * shape[1]), dtype=torch.float64)
    hk = dict(HK_SMALL, transformation=transformation)
    if transformation == 'flow':
        hp = O.make_hparams(**hk)
        params, _ = O.init_params(hp, (32, 32, 3), dtype=torch.float64)
        for k in params:
            if '/flows/' in k:
                params[k].zero_()                                          # zero flow everywhere
        inputs, noise = O.make_synthetic_inputs(hp, 2, (32, 32, 3), dtype=torch.float64)
        inputs['pix_distribs'] = const(hp, 2, (32, 32, 3))
        with torch.no_grad():
            out = P.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, 2))
    else:
        out = _oracle(hk, D=1, pix=const)[-1]
    for k in ('gen_pix_distribs', 'transformed_pix_distribs', 'gen_pix_distribs_enc'):
        assert (out[k] - 1.0 / 1024).abs().max() < 1e-15, k


@pytest.mark.parametrize('transformation', ['cdna', 'flow'])
def test_oracle_cell_step_pix_path_matches_a_numpy_loop(transformation):
    """One cell step's pix path restated with numpy loops from the reference lines, fed the step's own kernels / flows and
    masks, against the pix reference in fp64.  The flows the reference recomputes from the tap are the ones the oracle's
    step warped the image with."""
    hk = dict(HK_SMALL, nz=0, transformation=transformation)
    hp = O.make_hparams(**hk)
    H = W = 32
    params, _ = O.init_params(hp, (H, W, 3), dtype=torch.float64)
    if transformation == 'flow':
        params['generator/rnn/savp_cell/flows/conv2d/bias'] = torch.tensor([0.37, 1.27, -0.53, 2.17, 0.61, -1.41, 0.23, 1.79],
                                                                           dtype=torch.float64)
    inputs, _ = O.make_synthetic_inputs(hp, 2, (H, W, 3), dtype=torch.float64)
    pix = make_pix(hp, 2, H, W, 3)
    gen_prev = make_pix(hp, 2, H, W, 3, seed=7)[1]
    gt = torch.tensor([True, False])
    # zero recurrent states as generator_given_z builds them
    enc, dec = O.layer_specs(hp, H, W)
    rnn, hh = [], H
    for oc, use in enc:
        hh //= 2
        if use:
            rnn.append((torch.zeros(2, hh, hh, oc, dtype=torch.float64),) * 2)
    for oc, use in dec:
        hh *= 2
        if use:
            rnn.append((torch.zeros(2, hh, hh, oc, dtype=torch.float64),) * 2)
    states = dict(gen_image=inputs['images'][0] * 0.5, conv_rnn_states=rnn)
    tap = {}
    captured = {}
    real_warp = O.image_warp

    def warp(im, flow):                                                    # records the flows the step uses
        captured.setdefault('flows', []).append(flow)
        return real_warp(im, flow)
    O.image_warp = warp
    try:
        with torch.no_grad():
            out, _ = O.savp_cell_step(O.Vars(params), hp, 'generator/rnn/savp_cell', 1, dict(images=inputs['images'][1]),
                                      inputs['images'][0], states, gt, tap)
    finally:
        O.image_warp = real_warp
    flows = None
    if transformation == 'flow':
        flows = P.step_flows(O.Vars(params), hp, tap)
        for k in range(4):
            assert torch.equal(flows[..., k], captured['flows'][k])
    with torch.no_grad():
        gen, tr = P.pix_step(hp, pix[1], gen_prev, pix[0], gt, out['masks'][..., 0, :], kernels=tap['kernels'], flows=flows)
    masks = out['masks'][..., 0, :].numpy()                               # [B,H,W,L]
    p = np.where(gt.numpy()[:, None, None, None], pix[1].numpy(), gen_prev.numpy())
    first = pix[0].numpy()
    B, D, nk = 2, 3, 4
    want_t = np.zeros((B, H, W, D, nk + 3))
    for b in range(B):
        for y in range(H):
            for x in range(W):
                for k in range(nk):
                    if transformation == 'cdna':
                        kern = tap['kernels'].numpy()[b, :, :, k]
                        acc = np.zeros(D)
                        for i in range(5):
                            for j in range(5):
                                yy, xx = y + i - 2, x + j - 2
                                yy = -yy - 1 if yy < 0 else (2 * H - 1 - yy if yy >= H else yy)   # SYMMETRIC padding
                                xx = -xx - 1 if xx < 0 else (2 * W - 1 - xx if xx >= W else xx)
                                acc += kern[i, j] * p[b, yy, xx]
                    else:
                        fx, fy = captured['flows'][k][b, y, x].numpy()
                        x0, y0 = int(np.floor(fx)), int(np.floor(fy))
                        ax, ay = fx - x0, fy - y0
                        cx = lambda v: min(max(v, 0), W - 1)
                        cy = lambda v: min(max(v, 0), H - 1)
                        acc = ((1 - ax) * (1 - ay) * p[b, cy(y + y0), cx(x + x0)] + (1 - ax) * ay * p[b, cy(y + y0 + 1), cx(x + x0)]
                               + ax * (1 - ay) * p[b, cy(y + y0), cx(x + x0 + 1)] + ax * ay * p[b, cy(y + y0 + 1), cx(x + x0 + 1)])
                    want_t[b, y, x, :, k] = acc
                want_t[b, y, x, :, nk] = p[b, y, x]
                want_t[b, y, x, :, nk + 1] = first[b, y, x]
                want_t[b, y, x, :, nk + 2] = p[b, y, x]
    g = (want_t * masks[:, :, :, None, :]).sum(-1)
    want_g = g / g.sum(axis=(1, 2), keepdims=True)
    np.testing.assert_allclose(tr.numpy(), want_t, rtol=0, atol=1e-12)
    np.testing.assert_allclose(gen.numpy(), want_g, rtol=0, atol=1e-12)
