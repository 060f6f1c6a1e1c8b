"""CPU reference of the generator's layer choices `downsample_layer`, `upsample_layer` and `activation_layer`
(savp_model.py:394-397; ops.get_downsample_layer / get_upsample_layer / get_activation_layer, ops.py:1052-1098), built on
the SAVP oracle (oracle/savp_oracle.py) without changing it.

- downsample_layer='conv2d' (ops.conv2d, :494): a k x k convolution with stride 2, TF SAME padding and a bias, variables
  h{i}/conv2d/{kernel,bias} with the kernel [k, k, cin, oc] (k = 5 at h0, 3 elsewhere).
- upsample_layer='deconv2d' (ops.deconv2d, :553-590): tf.nn.conv2d_transpose with a 3x3 kernel, stride 2, SAME (output
  2H x 2W), plus a bias; variables h{i}/deconv2d/{kernel,bias} with the kernel [3, 3, oc, cin].
- conv_pool2d_v2 / upsample_conv2d_v2 (:859, :722) use the v1 variables and compute the v1 functions (ops.py:643-680,
  795-820; tests/test_layer_choices.py checks this in float64), so they run as v1 here.
- activation_layer='elu': tf.nn.elu at the h{i} sites and the h_flow / h_scratch / h_masks heads.  The posterior encoder
  keeps its leaky relu and the ConvLSTM cells their sigmoid / tanh.

For the duration of a call the oracle's variable store renames the h{i} variables (and transposes deconv2d's kernel
shape), the oracle's conv_pool2d / upsample_conv2d run the chosen layer for kernels that came from a renamed variable,
and the oracle's `torch.relu` applies the site activation to the tensors its normaliser produced (the CDNA kernels' relu
stays a relu).  The norm_layer and ConvLSTM variants of savp_norm_layer_oracle apply as well.  With the defaults every
function returns the result of savp_norm_layer_oracle."""
import re
from contextlib import contextmanager

import torch
import torch.nn.functional as F

import savp_norm_layer_oracle as NL
from oracle import savp_oracle as O

DOWN = re.compile(r'/h\d+/conv_pool2d/(kernel|bias)$')
UP = re.compile(r'/h\d+/upsample_conv2d/(kernel|bias)$')


def elu(x):
    """tf.nn.elu."""
    return torch.where(x > 0, x, torch.expm1(torch.clamp(x, max=0)))


def conv2d_s2(x, kernel, bias):
    """ops.conv2d(strides=2, padding='SAME') of x [N, H, W, Cin] with kernel [k, k, Cin, Cout]."""
    return O.conv2d_tf(x, kernel, strides=(2, 2), padding='SAME', bias=bias)


def deconv2d(x, kernel, bias):
    """ops.deconv2d(kernel_size=3, strides=2, padding='SAME'): tf.nn.conv2d_transpose of x [N, H, W, Cin] with kernel
    [3, 3, Cout, Cin] to [N, 2H, 2W, Cout] -- the adjoint of the 2H -> H SAME stride-2 conv, which pads 0 before and 1
    after, so output row 2 i + r receives input row i through tap r, and row 2H is cropped."""
    H, W = x.shape[1], x.shape[2]
    y = O._conv_op(lambda a, k: F.conv_transpose2d(a, k.permute(3, 2, 0, 1), stride=2), O._nchw(x), kernel)
    return O._nhwc(y[:, :, :2 * H, :2 * W]) + bias


def model_name(name, hp):
    """The model's name of an oracle variable under the layer choices."""
    if hp.downsample_layer == 'conv2d' and DOWN.search(name):
        return name.replace('/conv_pool2d/', '/conv2d/')
    if hp.upsample_layer == 'deconv2d' and UP.search(name):
        return name.replace('/upsample_conv2d/', '/deconv2d/')
    return name


class _Torch(object):
    """The torch module with `relu` replaced (the oracle's module global `torch` during a call)."""

    def __init__(self, relu):
        self.relu = relu

    def __getattr__(self, name):
        return getattr(torch, name)


@contextmanager
def variant(hp):
    assert hp.downsample_layer in ('conv_pool2d', 'conv_pool2d_v2', 'conv2d'), hp.downsample_layer
    assert hp.upsample_layer in ('upsample_conv2d', 'upsample_conv2d_v2', 'deconv2d'), hp.upsample_layer
    assert hp.activation_layer in ('relu', 'elu'), hp.activation_layer
    with NL.variant(hp):
        down = hp.downsample_layer == 'conv2d'
        up = hp.upsample_layer == 'deconv2d'
        if not (down or up or hp.activation_layer == 'elu'):
            yield
            return
        renamed = {}            # id -> kernel of a renamed h{i} variable (kept alive, so ids stay unique)
        normed = {}             # id -> output of a site normaliser (kept alive for the same reason)
        saved = O.Vars.get, O.conv_pool2d, O.upsample_conv2d, O.instance_norm, O.torch

        def get(self, name, shape, init='kernel', trainable=True):
            new = model_name(name, hp)
            if new != name and name.endswith('/upsample_conv2d/kernel'):
                shape = (shape[0], shape[1], shape[3], shape[2])
            p = saved[0](self, new, shape, init, trainable)
            if new != name:
                renamed[id(p)] = p
            return p

        def conv_pool2d(x, kernel, bias):
            return conv2d_s2(x, kernel, bias) if id(kernel) in renamed else saved[1](x, kernel, bias)

        def upsample_conv2d(x, kernel, bias):
            return deconv2d(x, kernel, bias) if id(kernel) in renamed else saved[2](x, kernel, bias)

        def instance_norm(x, gamma, beta, eps=1e-6):
            y = saved[3](x, gamma, beta, eps)
            normed[id(y)] = y
            return y

        def relu(x):
            return elu(x) if id(x) in normed else torch.relu(x)

        O.Vars.get, O.conv_pool2d, O.upsample_conv2d = get, conv_pool2d, upsample_conv2d
        if hp.activation_layer == 'elu':
            O.instance_norm, O.torch = instance_norm, _Torch(relu)
        try:
            yield
        finally:
            O.Vars.get, O.conv_pool2d, O.upsample_conv2d, O.instance_norm, O.torch = saved


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
    """O.init_params tracing the variant: conv2d / deconv2d variables and the norm_layer / ConvLSTM variants' variables."""
    with variant(hp):
        return O.init_params(hp, image_shape, batch, action_dim, seed, dtype)
