"""Cost of where and how the SAVP cell takes its conditioning vector at cfg2 (SAVP, 64x64x3, 2 + 10 frames, B = 16): the
default (tile-concat into every convolution) against where_add='input' (h0 alone), where_add='middle' (the first decoder
layer alone), use_tile_concat=False (dense(v) prefilled into every site's output), and use_tile_concat=False with the
norm-free generator and ConvLSTM (norm_layer='none', conv_rnn_norm_layer='none').  In alternating rounds: the median of --reps captured training steps and of --reps `generator_forward` calls,
timed with CUDA events.  Prints the card's name, power limit and SM clocks first, then one JSON line per row.
Usage: python tests/measure_conditioning.py [--reps N] [--rounds R] [--out FILE.json]"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from measure_conv_lstm import CONFIGS, card, time_model  # noqa: E402

CHOICES = [('default', {}), ('where_add_input', dict(where_add='input')), ('where_add_middle', dict(where_add='middle')),
           ('no_tile_concat', dict(use_tile_concat=False)),
           ('no_tile_concat_norm_free', dict(use_tile_concat=False, norm_layer='none', conv_rnn_norm_layer='none'))]


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
