"""Cost of the robot-state path: the training step of cfg2 (SAVP, 64x64x3, 2 + 10 frames, B = 16) with 4-dim actions, without
and with 3-dim states, alternated, timed with CUDA events on the captured step as bench.py runs it; the same for the cfg3
shape (2 + 28 frames, B = 32); the recurrence kernel (vp_state_pred_fwd) on its own; and the kernel launches of one eager
step.  Prints the card's name, power limit and SM clocks first, then one JSON line per measurement.
Usage: python tests/measure_states.py [--reps N] [--rounds R] [--configs cfg2_actions,cfg3_shape] [--out FILE.json]"""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from video_prediction_b200 import lib as L  # noqa: E402
from video_prediction_b200.models import get_model_class  # noqa: E402

SAVP = dict(lr=0.0002, beta1=0.5, beta2=0.999, l1_weight=100.0, l2_weight=0.0, kl_weight=1.0, video_sn_vae_gan_weight=0.1,
            video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, gan_feature_cdist_weight=0.0, state_weight=0.0)
CONFIGS = [('cfg2_actions', dict(SAVP, context_frames=2, sequence_length=12), 16),
           ('cfg3_shape', dict(SAVP, context_frames=2, sequence_length=30), 32)]
A, SD = 4, 3


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def batch(hk, B, sd):
    g = torch.Generator().manual_seed(0)
    T = hk['sequence_length']
    inp = {'images': torch.rand(B, T, 64, 64, 3, generator=g), 'actions': torch.randn(B, T - 1, A, generator=g)}
    if sd:
        inp['states'] = torch.randn(B, T, sd, generator=g)
    return inp


def time_steps(hk, B, sd, reps, warmup=3):
    """Median and min of `reps` captured training steps (resident inputs, fresh noise per step) + launches of the eager step."""
    model = get_model_class('savp')(mode='train', hparams_dict=hk)
    model.build_graph(batch(hk, B, sd))
    model.use_cuda_graph = True
    n0 = L.launch_count()
    model.train_step()                              # step 0 runs eagerly; the graph is captured on the next one
    torch.cuda.synchronize()
    launches = L.launch_count() - n0
    for _ in range(warmup):
        model.train_step()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        model.train_step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    kernel_ms = time_kernel(model, reps=200) if sd else None
    del model
    gc.collect()                                    # the layers refer back to the model: free its buffers before the next one
    torch.cuda.empty_cache()
    times.sort()
    return times[len(times) // 2], times[0], launches, kernel_ms


def time_kernel(model, reps):
    """vp_state_pred_fwd alone on the model's buffers: CUDA events around `reps` back-to-back launches."""
    model._state_pred_forward()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        model._state_pred_forward()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write every row to this JSON file')
    ap.add_argument('--configs', default=','.join(c[0] for c in CONFIGS), help='comma-separated subset of the configurations')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    for name, hk, B in [c for c in CONFIGS if c[0] in args.configs.split(',')]:
        for rnd in range(args.rounds):             # alternating: Sd = 0, 3, 0, 3, ...
            for sd in (0, SD):
                try:
                    med, best, launches, kms = time_steps(hk, B, sd, args.reps)
                except torch.cuda.OutOfMemoryError:
                    row = dict(config=name, B=B, Sd=sd, round=rnd, error='out of memory')
                    gc.collect()
                    torch.cuda.empty_cache()
                else:
                    row = dict(config=name, B=B, A=A, Sd=sd, round=rnd, step_ms_median=round(med, 3), step_ms_min=round(best, 3),
                               launches_per_eager_step=launches)
                    if kms is not None:
                        row['state_pred_kernel_us'] = round(kms * 1000, 2)
                rows.append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
