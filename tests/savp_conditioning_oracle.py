"""CPU reference of where and how the SAVP cell takes its conditioning vector state_action_z = [actions | state | rnn_z]
(savp_model.py:176-177, 436-518, 983-993; rnn_ops.py:128-146), built on the SAVP oracle (oracle/savp_oracle.py) without
changing it.

- where_add: 'all' feeds every h{i} convolution and every ConvLSTM / conv_h site; 'input' the h0 convolution alone; 'middle'
  the first decoder convolution h{n_enc} alone.  Under 'input' and 'middle' no ConvLSTM sees the vector (:467-473).
- use_tile_concat=True: the vector is tiled over space as extra input channels (ops.tile_concat).
- use_tile_concat=False (_maybe_tile_concat_layer, :983-993): the convolution reads the spatial input alone and
  dense(v, out_channels, use_bias=False) is added to its output, before the norm and the activation: `h{i}/dense/kernel`
  [Zc, oc] at an h{i} site, `conv_h{i}/dense/kernel` [Zc, oc] at an ablation_rnn site, and inside the ConvLSTM
  (BasicConv2DLSTMCell._dense) `lstm_h{i}/basic_conv2dlstm_cell/weights` [Zc, 4F] added to the gates' pre-activation before
  the cell's norm.  Without actions, states or z the reference's `concat` is a [B, 0] tensor, so the kernels are [0, oc].

For the duration of a call the oracle's `tile_concat_z` decides per site (the sites come in the order O.savp_cell_step
visits them: h{i}, then its ConvLSTM), and a site's dense term is added by wrapping the oracle's conv_pool2d /
upsample_conv2d (h{i} sites) or, during the ConvLSTM / conv_h call, its conv2d_tf.  The recurrence, norm_layer and ConvLSTM
variants of savp_recurrence_oracle apply as well, and inputs with 'states' run through savp_state_oracle.  With
where_add='all' and use_tile_concat=True every function returns exactly the oracle's result."""
from contextlib import contextmanager

import torch

import savp_recurrence_oracle as R
import savp_state_oracle as ST
from oracle import savp_oracle as O


def takes_vector(hp, li, rnn, n_enc):
    """Whether the h{li} convolution (rnn=False) or the ConvLSTM / conv_h site of layer li (rnn=True) gets the vector."""
    if rnn:
        return hp.where_add == 'all'                                                      # :467, :503
    return hp.where_add == 'all' or (hp.where_add == 'input' and li == 0) or (hp.where_add == 'middle' and li == n_enc)


def dense_kernel_name(hp, scope, li, rnn):
    if not rnn:
        return '%s/h%d/dense/kernel' % (scope, li)
    if hp.ablation_rnn:
        return '%s/conv_h%d/dense/kernel' % (scope, li)
    return '%s/lstm_h%d/basic_conv2dlstm_cell/weights' % (scope, li)


@contextmanager
def variant(hp):
    assert hp.where_add in ('input', 'all', 'middle'), hp.where_add
    with R.variant(hp):
        if hp.where_add == 'all' and hp.use_tile_concat:
            yield
            return
        saved = O.savp_cell_step, O.tile_concat_z, O.conv_pool2d, O.upsample_conv2d, O.conv_lstm_cell, O.conv2d_tf
        ctx = dict(sites=[], k=0, V=None, scope=None, n_enc=0)
        pending = {}        # id(site input) -> (dense kernel name, v, the input itself, kept alive so that ids stay unique)

        def savp_cell_step(V, hp_, scope, t, inp, first_image, states, ground_truth_t, tap=None):
            enc, dec = O.layer_specs(hp_, inp['images'].shape[1], inp['images'].shape[2])
            sites = []
            for li, (_, use) in enumerate(enc + dec):
                sites += [(li, False)] + ([(li, True)] if use else [])
            ctx.update(sites=sites, k=0, V=V, scope=scope, n_enc=len(enc))
            pending.clear()
            return saved[0](V, hp_, scope, t, inp, first_image, states, ground_truth_t, tap)

        def tile_concat_z(h, z):
            li, rnn = ctx['sites'][ctx['k']]
            ctx['k'] += 1
            if not takes_vector(hp, li, rnn, ctx['n_enc']):
                return h
            if hp.use_tile_concat:
                return saved[1](h, z)
            v = torch.zeros(h.shape[0], 0, dtype=h.dtype) if z is None else z      # concat([]) = zeros([B, 0]) (:436-438)
            x = h.view_as(h)
            pending[id(x)] = (dense_kernel_name(hp, ctx['scope'], li, rnn), v, x)
            return x

        def dense_term(name, v, c):
            return O.dense(v, ctx['V'].get(name, (v.shape[-1], c)))[:, None, None, :]

        def site(conv):
            def call(x, kernel, bias):
                y = conv(x, kernel, bias)
                if id(x) not in pending:
                    return y
                name, v, _ = pending.pop(id(x))
                return y + dense_term(name, v, y.shape[-1])
            return call

        def conv_lstm_cell(V, scope, inputs, state, filters):
            if id(inputs) not in pending:
                return saved[4](V, scope, inputs, state, filters)
            name, v, _ = pending.pop(id(inputs))

            def conv2d_tf(x, kernel, strides=(1, 1), padding='SAME', bias=None, tag=''):
                y = saved[5](x, kernel, strides, padding, bias, tag)
                return y + dense_term(name, v, y.shape[-1])           # rnn_ops.py:145-146, before the norm
            O.conv2d_tf = conv2d_tf
            try:
                return saved[4](V, scope, inputs, state, filters)
            finally:
                O.conv2d_tf = saved[5]

        O.savp_cell_step, O.tile_concat_z = savp_cell_step, tile_concat_z
        O.conv_pool2d, O.upsample_conv2d, O.conv_lstm_cell = site(saved[2]), site(saved[3]), conv_lstm_cell
        try:
            yield
        finally:
            O.savp_cell_step, O.tile_concat_z, O.conv_pool2d, O.upsample_conv2d, O.conv_lstm_cell, O.conv2d_tf = saved


def generator(V, hp, inputs, noise, ground_truth, taps=None):
    with variant(hp):
        if 'states' in inputs:
            return ST.generator(V, hp, inputs, noise, ground_truth, taps)
        return O.generator(V, hp, inputs, noise, ground_truth, taps)


def train_step(params, opt, hp, inputs, noise, step, sampling=None):
    with variant(hp):
        return ST.train_step(params, opt, hp, inputs, noise, step, sampling)


def init_params(hp, image_shape, batch=1, action_dim=0, state_dim=0, seed=0, dtype=torch.float32):
    """O.init_params tracing the sites' conditioning: fewer input channels where a site takes no tile-concat, the dense
    kernels, and the recurrence / norm variants' variables (state_pred with state_dim > 0)."""
    with variant(hp):
        return ST.init_params(hp, image_shape, batch, action_dim, state_dim, seed, dtype)
