"""CPU reference of the SAVP cell's recurrence choices (savp_model.py:263-307, 354-362, 424-434, 465-483, 500-517), built on
the SAVP oracle (oracle/savp_oracle.py) without changing it.

- ablation_rnn=True: every ConvLSTM becomes a stateless site in the scope `conv_h{i}`: conv2d 5x5 SAME with a bias
  (`conv2d/kernel` [5, 5, cin, oc], `conv2d/bias`), then norm_layer (`conv_h{i}/InstanceNorm` or `LayerNorm`, nothing for
  'none'), then activation_layer.  The z cell becomes `fc_z`: tanh(dense(z)) with `fc_z/dense/kernel` [nz, nz].
- rnn='gru': the z cell is tf.contrib.rnn.GRUCell(nz) (TF >= 1.9) in the scope `gru_z/gru_cell`:
  r, u = split(sigmoid([z, h] gates/kernel + gates/bias)), gates/bias initialised to ones;
  c = tanh([z, r h] candidate/kernel + candidate/bias);  h' = u h + (1 - u) c.  The state is h.
- use_rnn_z=False is a branch of the oracle itself (savp_cell_step): the zs go straight into the tile-concat vector.
- learn_initial_state=True: zero-initialised variables `generator/initial_state_{k}/initial_state`, tiled over the batch,
  replace the zero state entering step 0 (savp_model.py:295-307, 344-348).  k follows nest.flatten of
  {'conv_rnn_states': [(c, h) per ConvLSTM], 'rnn_z_state': (c, h) of lstm_z or h of gru_z}: the dict's keys sorted, so
  the ConvLSTMs first.  No ConvLSTM entries under ablation_rnn; no z entry without a z RNN (nz = 0, use_rnn_z=False or
  ablation_rnn), as the reference's state_size has none (:263-283).

For the duration of a call the oracle's `conv_lstm_cell` and `dense_lstm_cell` are swapped for the variant's cells (and
`savp_cell_step` for one that loads the learned initial states at t = 0); the
norm_layer and ConvLSTM variants of savp_norm_layer_oracle apply as well.  With the defaults every function returns the
oracle's result."""
from contextlib import contextmanager

import torch
import torch.nn.functional as F

import savp_norm_layer_oracle as NL
from oracle import savp_oracle as O


def conv_h_site(hp):
    """The ablation's conv_h{i} site, called where the oracle calls the ConvLSTM (scope .../lstm_h{i}/basic_conv2dlstm_cell):
    the state passes through untouched."""
    def cell(V, scope, inputs, state, filters):
        s = scope.rsplit('/', 2)[0] + '/conv_h' + scope.rsplit('/', 2)[1][len('lstm_h'):]
        k = V.get(s + '/conv2d/kernel', (5, 5, inputs.shape[-1], filters))
        b = V.get(s + '/conv2d/bias', (filters,), 'zeros')
        h = O.conv2d_tf(inputs, k, padding='SAME', bias=b)
        if hp.norm_layer != 'none':
            ns = s + ('/InstanceNorm' if hp.norm_layer == 'instance' else '/LayerNorm')
            g, be = V.get(ns + '/gamma', (filters,), 'ones'), V.get(ns + '/beta', (filters,), 'zeros')
            h = O.instance_norm(h, g, be) if hp.norm_layer == 'instance' else NL.layer_norm(h, g, be)
        h = F.elu(h) if hp.activation_layer == 'elu' else torch.relu(h)
        return h, state
    return cell


def fc_z_cell(V, scope, x, state, units):
    """savp_model.py:427-429: fc_z = tanh(dense(z)), no state."""
    s = scope.replace('/lstm_z/basic_lstm_cell', '/fc_z/dense')
    k = V.get(s + '/kernel', (x.shape[-1], units))
    b = V.get(s + '/bias', (units,), 'zeros')
    return torch.tanh(O.dense(x, k, b)), state


def gru_z_cell(V, scope, x, state, units):
    """GRUCell.call (TF >= 1.9); the oracle's (c, h) state tuple carries h in both slots."""
    s = scope.replace('/lstm_z/basic_lstm_cell', '/gru_z/gru_cell')
    h = state[1]
    wg = V.get(s + '/gates/kernel', (x.shape[-1] + units, 2 * units))
    bg = V.get(s + '/gates/bias', (2 * units,), 'ones')
    wc = V.get(s + '/candidate/kernel', (x.shape[-1] + units, units))
    bc = V.get(s + '/candidate/bias', (units,), 'zeros')
    r, u = torch.split(torch.sigmoid(torch.cat([x, h], dim=-1) @ wg + bg), units, dim=-1)
    c = torch.tanh(torch.cat([x, r * h], dim=-1) @ wc + bc)
    new_h = u * h + (1 - u) * c
    return new_h, (new_h, new_h)


def initial_state_step(step):
    """savp_cell_step with the learned initial states in place of the zero state at t = 0 (SAVPCell.zero_state)."""
    def call(V, hp, scope, t, inp, first_image, states, ground_truth_t, tap=None):
        if t == 0:
            B, k = inp['images'].shape[0], [0]

            def var(shape):
                v = V.get('generator/initial_state_%d/initial_state' % k[0], tuple(shape), 'zeros')
                k[0] += 1
                return v[None].expand((B,) + tuple(shape))
            states = dict(states)
            if not hp.ablation_rnn:
                states['conv_rnn_states'] = [(var(c.shape[1:]), var(h.shape[1:])) for c, h in states['conv_rnn_states']]
            if 'zs' in inp and hp.use_rnn_z and not hp.ablation_rnn:
                if hp.rnn == 'lstm':
                    states['rnn_z_state'] = (var((hp.nz,)), var((hp.nz,)))
                else:
                    h = var((hp.nz,))
                    states['rnn_z_state'] = (h, h)
        return step(V, hp, scope, t, inp, first_image, states, ground_truth_t, tap)
    return call


@contextmanager
def variant(hp):
    # conv_rnn, conv_rnn_norm_layer and ablation_conv_rnn_norm have no effect under ablation_rnn (the cell is replaced)
    base = O.make_hparams(**dict(hp, conv_rnn_norm_layer='instance', ablation_conv_rnn_norm=False)) \
        if hp.ablation_rnn else hp
    with NL.variant(base):
        saved = O.conv_lstm_cell, O.dense_lstm_cell, O.savp_cell_step
        if hp.ablation_rnn:
            O.conv_lstm_cell, O.dense_lstm_cell = conv_h_site(hp), fc_z_cell
        elif hp.rnn == 'gru':
            O.dense_lstm_cell = gru_z_cell
        if hp.learn_initial_state:
            O.savp_cell_step = initial_state_step(O.savp_cell_step)
        try:
            yield
        finally:
            O.conv_lstm_cell, O.dense_lstm_cell, O.savp_cell_step = saved


def savp_cell_step(V, hp, scope, t, inp, first_image, states, ground_truth_t, tap=None):
    with variant(hp):
        return O.savp_cell_step(V, hp, scope, t, inp, first_image, states, ground_truth_t, tap)


def generator(V, hp, inputs, noise, ground_truth, taps=None):
    with variant(hp):
        return O.generator(V, hp, inputs, noise, ground_truth, taps)


def train_step(params, opt, hp, inputs, noise, step, sampling=None):
    with variant(hp):
        return O.train_step(params, opt, hp, inputs, noise, step, sampling)


def init_params(hp, image_shape, batch=1, action_dim=0, seed=0, dtype=torch.float32):
    """O.init_params tracing the variant's cells: conv_h{i} and fc_z, or gru_z, instead of the LSTMs' variables, and the
    learned initial states."""
    with variant(hp):
        return O.init_params(hp, image_shape, batch, action_dim, seed, dtype)
