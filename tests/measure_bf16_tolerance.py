"""bf16-vs-tolerance measurement (VERDICT round 1, item 7), done on the CPU oracle: the generator forward of cfg2 (SAVP 64x64,
2 context + 10 predicted frames) and of the 30-frame cfg3 shape with the convolution operands quantised as a tensor core
would read them -- TF32 as the CUDA path does (activations truncated, weights rounded to nearest) and bf16 (what kind::f16
operands would see) -- against the un-quantised fp32 oracle.  The contract is 1e-3 max-abs on images in [0, 1].
Usage: python tests/measure_bf16_tolerance.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import savp_oracle as O  # noqa: E402

torch.set_num_threads(16)
CASES = [('cfg2 SAVP 64x64x3, T = 12, nz = 8', dict(context_frames=2, sequence_length=12, nz=8), 2, (64, 64, 3), 0),
         ('cfg3 shape 64x64x3, T = 30, nz = 8, 4 actions', dict(context_frames=2, sequence_length=30, nz=8), 2, (64, 64, 3), 4)]
for name, hk, B, shape, A in CASES:
    hp = O.make_hparams(**hk)
    params, _ = O.init_params(hp, shape, action_dim=A, seed=0)
    inputs, noise = O.make_synthetic_inputs(hp, B, shape, action_dim=A, seed=0)
    outs = {}
    for tag, mode, wmode in (('fp32', None, 'rna'), ('tf32', 'trunc', 'rna'), ('bf16', 'bf16', 'bf16')):
        O.set_tf32_emulation(mode, weight_mode=wmode)
        with torch.no_grad():
            outs[tag] = O.generator(O.Vars(params), hp, inputs, noise, O.ground_truth_mask(hp, B))['gen_images']
    O.set_tf32_emulation(None)
    print(name)
    for tag in ('tf32', 'bf16'):
        d = (outs[tag] - outs['fp32']).abs()
        per_t = d.flatten(1).max(dim=1).values
        print('  %s operands vs fp32: max-abs %.2e (tolerance 1e-3: %s), mean-abs %.2e, max-abs per predicted frame first/last %.2e / %.2e'
              % (tag, d.max().item(), 'inside' if d.max().item() <= 1e-3 else 'OUTSIDE', d.mean().item(), per_t[0].item(), per_t[-1].item()))
