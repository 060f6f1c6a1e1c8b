"""CPU reference of the robot-state path of the action-conditioned SAVP cell (savp_model.py:411-421, 655-658, 666-667,
684-685), built on the SAVP oracle (oracle/savp_oracle.py) without changing it.

Per step t the cell selects state_t = ground_truth[t] ? states[t] : gen_state_{t-1} (the zero state before the first step),
tile-concatenates [actions_t | stop_gradient(state_t) | rnn_z_t] into every convolution input, and predicts
gen_state_t = dense([actions_t | state_t]) under `state_pred`.  The states read no image, so `generator_given_z` runs the
recurrence first and hands the oracle's own unroll the conditioning vector [actions_t | state_t] in place of the actions:
the oracle then concatenates [that | rnn_z] at every tile-concat site, which is the reference's order.  The posterior
encoder still sees the actions alone (savp_model.py:21-51).  Inputs are time-major as the oracle's: states [T,B,Sd]."""
from collections import OrderedDict
from contextlib import contextmanager

import numpy as np
import torch

from oracle import savp_oracle as O

SCOPE = 'generator/rnn/savp_cell'


def state_pred(V, action, state, scope=SCOPE):
    """gen_state = dense([action | state]) (savp_model.py:655-658; ops.dense, ops.py:5-16)."""
    x = state if action is None else torch.cat([action, state], dim=-1)
    sd = state.shape[-1]
    k = V.get(scope + '/state_pred/dense/kernel', (x.shape[-1], sd))
    b = V.get(scope + '/state_pred/dense/bias', (sd,), 'zeros')
    return O.dense(x, k, b)


def _condition(action, state):
    """The tile-concat vector without rnn_z: [actions | stop_gradient(state)] (savp_model.py:414-421)."""
    return state.detach() if action is None else torch.cat([action, state.detach()], dim=-1)


def savp_cell_step(V, hp, scope, t, inp, first_image, rnn_states, ground_truth_t, tap=None):
    """O.savp_cell_step with inp['states'] [B,Sd], the ground-truth robot state of step t.  rnn_states is the oracle's cell
    state plus 'gen_state' [B,Sd], the previous prediction.  Returns the oracle's outputs + gen_states, and the new state."""
    B = inp['images'].shape[0]
    state = torch.where(ground_truth_t.view(B, 1), inp['states'], rnn_states['gen_state'])     # :411-412
    action = inp.get('actions')
    plain = {k: v for k, v in inp.items() if k != 'states'}
    plain['actions'] = _condition(action, state)
    out, new = O.savp_cell_step(V, hp, scope, t, plain, first_image, rnn_states, ground_truth_t, tap)
    gen_state = state_pred(V, action, state, scope)                                              # after the masks, as :655
    out['gen_states'] = gen_state
    new['gen_state'] = gen_state
    return out, new


def generator_given_z(V, hp, inputs, ground_truth, scope=SCOPE, taps=None):
    """O.generator_given_z + the states.  inputs as the oracle's, plus states [T,B,Sd]."""
    if 'states' not in inputs:
        return O.generator_given_z(V, hp, inputs, ground_truth, scope=scope, taps=taps)
    states = inputs['states']
    gen = torch.zeros_like(states[0])            # zero_state of gen_state; never read, ground_truth[0] is True (context)
    conds, gens = [], []
    for t in range(hp.sequence_length - 1):
        action = inputs['actions'][t] if 'actions' in inputs else None
        state = torch.where(ground_truth[t].view(-1, 1), states[t], gen)
        gen = state_pred(V, action, state, scope)
        conds.append(_condition(action, state))
        gens.append(gen)
    plain = {k: v for k, v in inputs.items() if k != 'states'}
    plain['actions'] = torch.stack(conds)
    out = O.generator_given_z(V, hp, plain, ground_truth, scope=scope, taps=taps)
    out['gen_states'] = torch.stack(gens)
    return out


def generator(V, hp, inputs, noise, ground_truth, taps=None):
    """O.generator (generator_fn, savp_model.py:699-768) + the states of both unrolls (gen_states, gen_states_enc)."""
    if hp.nz == 0:
        return generator_given_z(V, hp, inputs, ground_truth, taps=taps)
    z_mu, z_lss = O.posterior(V, hp, inputs)                                  # actions only (:21-51)
    zs_post = z_mu + torch.sqrt(torch.exp(z_lss)) * noise['eps']             # :712
    zs_prior = torch.cat([zs_post[:hp.context_frames - 1], noise['z_prior']], dim=0)   # :724-725
    out_enc = generator_given_z(V, hp, dict(inputs, zs=zs_post), ground_truth)          # :730
    out = generator_given_z(V, hp, dict(inputs, zs=zs_prior), ground_truth, taps=taps)  # :732
    outputs = OrderedDict(out)
    outputs['zs_mu_enc'] = z_mu
    outputs['zs_log_sigma_sq_enc'] = z_lss
    for k, v in out_enc.items():
        outputs[k + '_enc'] = v
    return outputs


@contextmanager
def _oracle_generator(fn):
    """O.train_step and O.init_params look `generator` up in their module when they run: swap in `fn` meanwhile."""
    saved = O.generator
    O.generator = fn
    try:
        yield
    finally:
        O.generator = saved


def train_step(params, opt, hp, inputs, noise, step, sampling=None):
    """O.train_step with the states generator.  No loss reads gen_states, so state_pred gets no gradient (None)."""
    if 'states' not in inputs:
        return O.train_step(params, opt, hp, inputs, noise, step, sampling)
    with _oracle_generator(generator):
        return O.train_step(params, opt, hp, inputs, noise, step, sampling)


def init_params(hp, image_shape, batch=1, action_dim=0, state_dim=0, seed=0, dtype=torch.float32):
    """O.init_params, tracing the states generator when state_dim > 0 (creates state_pred/dense/{kernel,bias})."""
    if not state_dim:
        return O.init_params(hp, image_shape, batch, action_dim, seed, dtype)
    zeros = torch.zeros(hp.sequence_length, batch, state_dim, dtype=dtype)

    def traced(V, hp_, inputs, noise, gt, taps=None):
        return generator(V, hp_, dict(inputs, states=zeros), noise, gt, taps)
    with _oracle_generator(traced):
        return O.init_params(hp, image_shape, batch, action_dim, seed, dtype)


def make_synthetic_inputs(hp, batch, image_shape, action_dim=0, state_dim=0, seed=0, dtype=torch.float32, smooth=True):
    """O.make_synthetic_inputs (unchanged values) + states [T,B,state_dim] ~ N(0,1) from a generator of their own."""
    inputs, noise = O.make_synthetic_inputs(hp, batch, image_shape, action_dim, seed, dtype, smooth)
    if state_dim:
        rng = np.random.default_rng(seed + 2000)
        inputs['states'] = torch.tensor(rng.standard_normal((hp.sequence_length, batch, state_dim)), dtype=dtype)
    return inputs, noise
