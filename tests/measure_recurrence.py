"""Cost of the recurrence ablation (ablation_rnn: each ConvLSTM becomes a 5x5 conv + instance norm + relu, the z LSTM a dense
+ tanh) against the default model, cfg2 (SAVP, 64x64x3, 2 + 10 frames, B = 16), in alternating rounds: the median captured
training step and the median `generator_forward`, timed with CUDA events.  Then each conv_h convolution of the cfg2 ablated
generator alone (NB = 2B), CUDA events around back-to-back engine launches, with TFLOP/s from the algorithmic FLOPs and the
share of the H100 SXM data-sheet dense TF32 rate (495 TFLOP/s; a power-limited card reaches less).  Prints the card's name,
power limit and SM clocks first, then one JSON line per row.
Usage: python tests/measure_recurrence.py [--reps N] [--rounds R] [--out FILE.json]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from measure_conv_lstm import CONFIGS, card, time_model  # noqa: E402
from video_prediction_b200 import lib as L  # noqa: E402

TF32_PEAK = 495e12
VARIANTS = [('default', {}), ('ablation_rnn', dict(ablation_rnn=True))]


def time_conv_h(B, reps=50):
    """Each conv_h{i} forward of the cfg2 ablated generator: (h{i} | z) -> oc, 5x5 stride 1, NB = 2B."""
    rows = []
    nb = 2 * B
    for hw, oc in ((32, 32), (16, 64), (8, 128)):
        ci = oc + 8
        gen = torch.Generator().manual_seed(oc)
        x = torch.randn(nb, hw, hw, ci, generator=gen).cuda()
        w = (torch.randn(5, 5, ci, oc, generator=gen) * 0.03).cuda()
        bias = torch.zeros(oc, device='cuda')
        y = torch.empty(nb, hw, hw, oc, device='cuda')
        wp, n_pad, kc = L.pack_weights(w, (1, 5, 5), ci, oc, L.WKIND_PLAIN, L.WLAYOUT_FWD)
        g = L.geom((1, 5, 5), (1, 1, 1), (0, 2, 2))
        xv, yv = L.tensor_view(x, ci), L.tensor_view(y)
        fn = lambda: L.conv_igemm(xv, g, wp, n_pad, kc, yv, bias)      # noqa: E731
        flops = 2.0 * nb * hw * hw * oc * ci * 25
        ts = []
        for _ in range(3):
            fn()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b) / reps)
        t = sorted(ts)[1]
        rate = flops / (t * 1e-3)
        rows.append(dict(layer='conv_h %dx%d oc=%d ci=%d NB=%d' % (hw, hw, oc, ci, nb), gflop=round(flops / 1e9, 3),
                         us=round(t * 1000, 2), tflops=round(rate / 1e12, 1), tf32_peak_share=round(rate / TF32_PEAK, 3)))
    return rows


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
        for vname, v in VARIANTS:
            step, fwd = time_model(dict(hk, **v), B, args.reps)
            row = dict(config=name, B=B, variant=vname, round=rnd, step_ms_median=round(step, 3),
                       generator_forward_ms_median=round(fwd, 3))
            rows.append(row)
            print(json.dumps(row), flush=True)
    for row in time_conv_h(B):
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
