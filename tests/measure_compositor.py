"""Cost of the compositing hparams at cfg2 (SAVP, 64x64x3, 2 + 10 frames, B = 16): the default layers (4 CDNA transforms,
previous and first image, scratch image: 7 slots) against last_frames=2 (11 slots), the flow transforms of two frames, the
context images with the last-context image as backgrounds and independent masks, and the previous image alone (1 slot,
no heads).  In alternating rounds: the median of --reps captured training steps and of --reps `generator_forward` calls,
timed with CUDA events.  Prints the card's name, power limit and SM clocks first, then one JSON line per row.
Usage: python tests/measure_compositor.py [--reps N] [--rounds R] [--out FILE.json]"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from measure_conv_lstm import CONFIGS, card, time_model  # noqa: E402

CHOICES = [('default', {}), ('last_frames_2', dict(last_frames=2)),
           ('flow_last_frames_2', dict(transformation='flow', last_frames=2)),
           ('context_backgrounds_independent', dict(context_images_background=True, last_context_image_background=True,
                                                    dependent_mask=False)),
           ('prev_image_only', dict(num_transformed_images=0, first_image_background=False, generate_scratch_image=False))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None, help='also write every row to this JSON file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    name, hk, B = CONFIGS[0]
    for rnd in range(args.rounds):
        for choice, ch in CHOICES:
            step, fwd = time_model(dict(hk, **ch), B, args.reps)
            row = dict(config=name, B=B, choice=choice, round=rnd, step_ms_median=round(step, 3), generator_forward_ms_median=round(fwd, 3))
            rows.append(row)
            print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
