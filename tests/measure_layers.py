"""Cost of the generator's layer choices: the defaults (conv_pool2d, upsample_conv2d, relu) against
downsample_layer='conv2d', upsample_layer='deconv2d', activation_layer='elu' and all three together.  For cfg2 (SAVP,
64x64x3, 2 + 10 frames, B = 16), in alternating rounds: the median of --reps captured training steps and of --reps
`generator_forward` calls, timed with CUDA events.  Then every h{i} engine call of the cfg2 model alone, for the default layer and
the new one at the same site: forward (NB = 32 samples, one step), dgrad and wgrad (all 11 steps stacked, as the backward
runs them), CUDA events around --call-reps back-to-back launches (middle of three windows), TFLOP/s from the multiply-adds the geometry executes (2 x outputs x
taps per output x ci x co; a transposed stride-2 call executes taps / 4 per output).  Prints the card's name, power limit
and SM clocks first, then one JSON line per row.
Usage: python tests/measure_layers.py [--reps N] [--call-reps N] [--rounds R] [--out FILE.json]"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from measure_conv_lstm import CONFIGS, L, card, time_model  # noqa: E402

CHOICES = [('default', {}), ('conv2d', dict(downsample_layer='conv2d')), ('deconv2d', dict(upsample_layer='deconv2d')),
           ('both', dict(downsample_layer='conv2d', upsample_layer='deconv2d')), ('elu', dict(activation_layer='elu')),
           ('all3', dict(downsample_layer='conv2d', upsample_layer='deconv2d', activation_layer='elu'))]
NB, S = 32, 11
# (site, layer, kind, k, stride-2 pad before, transposed, ci (tile-concat included, padded to 4), co, input extent) of cfg2
SITES = [('h0', 'conv_pool2d', L.WKIND_POOLED, 5, 2, False, 16, 32, 64), ('h0', 'conv2d', L.WKIND_PLAIN, 5, 1, False, 16, 32, 64),
         ('h1', 'conv_pool2d', L.WKIND_POOLED, 3, 1, False, 40, 64, 32), ('h1', 'conv2d', L.WKIND_PLAIN, 3, 0, False, 40, 64, 32),
         ('h2', 'conv_pool2d', L.WKIND_POOLED, 3, 1, False, 72, 128, 16), ('h2', 'conv2d', L.WKIND_PLAIN, 3, 0, False, 72, 128, 16),
         ('h3', 'upsample_conv2d', L.WKIND_UPSAMPLED, 3, 2, True, 136, 64, 8), ('h3', 'deconv2d', L.WKIND_DECONV, 3, 0, True, 136, 64, 8),
         ('h4', 'upsample_conv2d', L.WKIND_UPSAMPLED, 3, 2, True, 136, 32, 16), ('h4', 'deconv2d', L.WKIND_DECONV, 3, 0, True, 136, 32, 16),
         ('h5', 'upsample_conv2d', L.WKIND_UPSAMPLED, 3, 2, True, 72, 32, 32), ('h5', 'deconv2d', L.WKIND_DECONV, 3, 0, True, 72, 32, 32)]


def _per_call_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def time_engine(reps):
    rows = []
    for site, layer, kind, k, pad, transposed, ci, co, e in SITES:
        ke = (1, k + 1, k + 1) if kind == L.WKIND_POOLED else ((1, k + 3, k + 3) if kind == L.WKIND_UPSAMPLED else (1, k, k))
        oe = 2 * e if transposed else e // 2
        wshape = (k, k, co, ci) if kind == L.WKIND_DECONV else (k, k, ci, co)
        gen = torch.Generator().manual_seed(k + ci)
        w = (torch.randn(*wshape, generator=gen) * 0.05).cuda()
        wp, n_pad, kc = L.pack_weights(w, (1, k, k), ci, co, kind, L.WLAYOUT_FWD)
        wpd, n_pad_d, kc_d = L.pack_weights(w, (1, k, k), ci, co, kind, L.WLAYOUT_DGRAD)
        g = L.geom(ke, (1, 2, 2), (0, pad, pad), transposed)
        gt = L.geom(ke, (1, 2, 2), (0, pad, pad), not transposed)
        x = torch.randn(S * NB, e, e, ci, generator=gen).cuda()
        dy = torch.randn(S * NB, oe, oe, co, generator=gen).cuda()
        out, dx = torch.empty(NB, oe, oe, co, device='cuda'), torch.empty(S * NB, e, e, ci, device='cuda')
        dwp = torch.zeros_like(wp)
        bias = torch.zeros(co, device='cuda')
        taps = ke[1] * ke[2] / (4.0 if transposed else 1.0)         # per output of the forward
        taps_d = ke[1] * ke[2] / (1.0 if transposed else 4.0)       # per output of the dgrad (the flipped geometry)
        flops = {'fwd': 2.0 * NB * oe * oe * co * ci * taps, 'dgrad': 2.0 * S * NB * e * e * ci * co * taps_d,
                 'wgrad': 2.0 * S * NB * oe * oe * co * ci * taps}
        calls = {
            'fwd': lambda: L.conv_igemm(L.tensor_view(x[:NB], ci), g, wp, n_pad, kc, L.tensor_view(out, co), bias, L.ACT_RELU),
            'dgrad': lambda: L.conv_igemm(L.tensor_view(dy, co), gt, wpd, n_pad_d, kc_d, L.tensor_view(dx, ci)),
            'wgrad': lambda: L.conv_wgrad(L.tensor_view(x, ci), L.tensor_view(dy, co), g, dwp, n_pad, kc, 0),
        }
        res = {}
        for _ in range(3):
            for name, fn in calls.items():
                res.setdefault(name, []).append(_per_call_ms(fn, reps))
        row = dict(site=site, layer=layer, geometry='%dx%d s2 pad %d%s' % (ke[1], ke[2], pad, ' transposed' if transposed else ''),
                   taps_per_output=taps, ci=ci, co=co, extent=e)
        for name, ts in res.items():
            t = sorted(ts)[1]
            row[name + '_us'] = round(t * 1000, 2)
            row[name + '_TFLOPs'] = round(flops[name] / (t * 1e-3) / 1e12, 1)
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--call-reps', type=int, default=100, help='launches per timing window of one engine call')
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None, help='also write every row to this JSON file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    for row in time_engine(args.call_reps):
        rows.append(row)
        print(json.dumps(row), flush=True)
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
