"""CPU reference of the generator's normaliser choice `norm_layer` (savp_model.py:394, ops.get_norm_layer ops.py:1062-1073),
built on the SAVP oracle (oracle/savp_oracle.py) without changing it.

norm_layer='layer' is tf.contrib.layers.layer_norm with its defaults, as TF 1.x defines it (its source is not part of the
reference tree):
- begin_norm_axis=1: mean and biased variance (tf.nn.moments) over H, W and C of each sample;
- begin_params_axis=-1: beta and gamma of shape [C], initialised to zeros and ones;
- variance_epsilon = 1e-12 for float32;
- y = gamma * (x - mean) * rsqrt(var + 1e-12) + beta, then the site's activation: relu in the generator, leaky relu 0.2
  in the posterior encoder;
- the variables live under the default scope `LayerNorm`, e.g. generator/rnn/savp_cell/h0/LayerNorm/gamma and
  generator/encoder/layer_2/LayerNorm/beta, in place of .../InstanceNorm/....
norm_layer='none' is tf.identity: the site computes act(conv + bias) and has no norm variables.

The sites are the normalised convolutions outside the ConvLSTM cells: h{i} (savp_model.py:463, 499), h{nl}_flow,
h{nl}_scratch and h{nl}_masks (:525, 564, 627) and the posterior encoder's layer_2.. (networks.py:12-27).  The norms of
the ConvLSTM cell, and the ablation's lstm_h{i}/InstanceNorm, follow conv_rnn_norm_layer and stay instance norms.

For the duration of a call the oracle's variable store renames the site variables to LayerNorm (or, for 'none', hands out
a marker instead of creating them), and the oracle's `instance_norm` applies layer norm to tensors that came from a
LayerNorm site and the identity to the marker.  The ConvLSTM variants of savp_conv_lstm_oracle are applied as well, so a
layer-norm generator with the norm-free cell is one call.  With norm_layer='instance' every function returns the result
of savp_conv_lstm_oracle, and so of the oracle itself for the default cell."""
import re
from contextlib import contextmanager

import torch

import savp_conv_lstm_oracle as CL
from oracle import savp_oracle as O

LN_EPS = 1e-12
SITE = re.compile(r'/(h\d+(_flow|_scratch|_masks)?|layer_\d+)/InstanceNorm/(gamma|beta)$')
NO_NORM = object()       # what a site's variable lookup returns with norm_layer='none'


def layer_norm(x, gamma, beta, eps=LN_EPS):
    """tf.contrib.layers.layer_norm(begin_norm_axis=1, begin_params_axis=-1) of x [N, ..., C]."""
    dims = tuple(range(1, x.dim()))
    mean = x.mean(dim=dims, keepdim=True)
    var = ((x - mean) ** 2).mean(dim=dims, keepdim=True)
    return (x - mean) * torch.rsqrt(var + eps) * gamma + beta


def site_name(name, norm_layer):
    """The model's name of an oracle variable: site norms move to the LayerNorm scope (None: no variable)."""
    if norm_layer == 'instance' or not SITE.search(name):
        return name
    return name.replace('/InstanceNorm/', '/LayerNorm/') if norm_layer == 'layer' else None


@contextmanager
def variant(hp):
    assert hp.norm_layer in ('instance', 'layer', 'none'), hp.norm_layer
    with CL.variant(hp):
        if hp.norm_layer == 'instance':
            yield
            return
        layer_gammas = set()       # ids of the gamma tensors of LayerNorm sites, alive for the whole call
        saved_get, saved_norm = O.Vars.get, O.instance_norm

        def get(self, name, shape, init='kernel', trainable=True):
            renamed = site_name(name, hp.norm_layer)
            if renamed is None:
                return NO_NORM
            p = saved_get(self, renamed, shape, init, trainable)
            if renamed != name:
                layer_gammas.add(id(p))
            return p

        def instance_norm(x, gamma, beta, eps=1e-6):
            if gamma is NO_NORM:
                return x
            if id(gamma) in layer_gammas:
                return layer_norm(x, gamma, beta)
            return saved_norm(x, gamma, beta, eps)

        O.Vars.get, O.instance_norm = get, instance_norm
        try:
            yield
        finally:
            O.Vars.get, O.instance_norm = saved_get, saved_norm


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
    """O.init_params tracing the variant: LayerNorm site variables, or none, and the ConvLSTM variant's variables."""
    with variant(hp):
        return O.init_params(hp, image_shape, batch, action_dim, seed, dtype)
