"""Cost of the pixel-distribution path: generator_forward time with D = 0, 1 and 2 designated pixels, at cfg2 (SAVP, B = 16)
and at a planning-sized action-conditioned batch (B = 128), timed with CUDA events.  Prints the card name and power limit
first, then one JSON line per measurement.  Usage: python tests/measure_pix_distribs.py [--reps N] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from video_prediction_b200.models import get_model_class  # noqa: E402

CONFIGS = [('cfg2_B16', dict(context_frames=2, sequence_length=12, nz=8), 16, 0),
           ('planning_B128_actions', dict(context_frames=2, sequence_length=12, nz=8), 128, 4)]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def time_forward(hk, B, A, D, reps, warmup=3):
    g = torch.Generator().manual_seed(0)
    inp = {'images': torch.rand(B, hk['sequence_length'], 64, 64, 3, generator=g)}
    if A:
        inp['actions'] = torch.randn(B, hk['sequence_length'] - 1, A, generator=g)
    if D:
        p = torch.rand(B, hk['sequence_length'], 64, 64, D, generator=g)
        inp['pix_distribs'] = p / p.sum(dim=(2, 3), keepdim=True)
    model = get_model_class('savp')(mode='test', hparams_dict=hk)
    model.build_graph(inp)
    model.set_inputs(inp)
    for _ in range(warmup):
        model.generator_forward(collect=False)
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        model.generator_forward(collect=False)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    del model
    torch.cuda.empty_cache()
    times.sort()
    return times[len(times) // 2], times[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None, help='also write every row to this JSON file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    for name, hk, B, A in CONFIGS:
        base = None
        for rnd in range(2):                       # two alternating rounds: D = 0, 1, 2, 0, 1, 2
            for D in (0, 1, 2):
                med, best = time_forward(hk, B, A, D, args.reps)
                if D == 0 and base is None:
                    base = med
                row = dict(config=name, B=B, D=D, round=rnd, forward_ms_median=round(med, 3), forward_ms_min=round(best, 3),
                           overhead_vs_D0_first_round=round(med / base - 1, 4))
                rows.append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
