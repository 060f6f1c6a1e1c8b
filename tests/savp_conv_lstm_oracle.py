"""CPU reference of the norm-free ConvLSTM forms of the SAVP cell (savp_model.py:364-391), built on the SAVP oracle
(oracle/savp_oracle.py) without changing it.

- conv_rnn_norm_layer='none': BasicConv2DLSTMCell with normalizer_fn=None (rnn_ops.py:115-126, 137-171).  The gate
  convolution has a bias `basic_conv2dlstm_cell/bias` [4F] and nothing is normalised:
  c' = c sigmoid(f + 1) + sigmoid(i) tanh(j),  h = tanh(c') sigmoid(o).
- ablation_conv_rnn_norm=True (with 'instance'): the same cell, and the layer's output is IN(h) under
  `lstm_h{i}/InstanceNorm` (savp_model.py:380-383); the recurrent state keeps the raw h.

For the duration of a call the oracle's `conv_lstm_cell` is swapped for the variant's cell; every other function of the
oracle runs unchanged.  With conv_rnn_norm_layer='instance' and no ablation every function returns the oracle's result."""
from contextlib import contextmanager

import torch

from oracle import savp_oracle as O


def plain_conv_lstm_cell(V, scope, inputs, state, filters):
    """BasicConv2DLSTMCell.call with normalizer_fn=None: the convolution gets a bias, no norm (rnn_ops.py:115-126)."""
    c, h = state
    args = torch.cat([inputs, h], dim=-1)                                    # rnn_ops.py:143
    kernel = V.get(scope + '/kernel', (5, 5, args.shape[-1], 4 * filters))   # :118-120
    bias = V.get(scope + '/bias', (4 * filters,), 'zeros')                   # :122-125
    concat = O.conv2d_tf(args, kernel, padding='SAME', bias=bias)
    i, j, f, o = torch.split(concat, filters, dim=-1)                        # :150
    new_c = c * torch.sigmoid(f + 1.0) + torch.sigmoid(i) * torch.tanh(j)    # :157-162
    new_h = torch.tanh(new_c) * torch.sigmoid(o)                             # :165
    return new_h, (new_c, new_h)


def ablation_conv_lstm_cell(V, scope, inputs, state, filters):
    """savp_model.py:380-383: the norm-free cell, then the layer's instance norm on h in the `lstm_h{i}` scope."""
    h, new_state = plain_conv_lstm_cell(V, scope, inputs, state, filters)
    ns = scope.rsplit('/', 1)[0] + '/InstanceNorm'                         # layers/normalization.py:94
    gamma = V.get(ns + '/gamma', (filters,), 'ones')
    beta = V.get(ns + '/beta', (filters,), 'zeros')
    return O.instance_norm(h, gamma, beta), new_state


def cell_for(hp):
    if hp.conv_rnn_norm_layer == 'none':
        assert not hp.ablation_conv_rnn_norm, 'the reference calls None(h) here'
        return plain_conv_lstm_cell
    assert hp.conv_rnn_norm_layer == 'instance'
    return ablation_conv_lstm_cell if hp.ablation_conv_rnn_norm else O.conv_lstm_cell


@contextmanager
def variant(hp):
    """O.savp_cell_step looks `conv_lstm_cell` up in its module when it runs: swap in the variant's cell meanwhile."""
    saved = O.conv_lstm_cell
    O.conv_lstm_cell = cell_for(hp)
    try:
        yield
    finally:
        O.conv_lstm_cell = saved


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
    """O.init_params tracing the variant's cell: basic_conv2dlstm_cell/bias and, for the ablation, lstm_h{i}/InstanceNorm."""
    with variant(hp):
        return O.init_params(hp, image_shape, batch, action_dim, seed, dtype)
