"""Cost of the generator's normaliser choice: norm_layer = 'instance' (the default), 'layer' and 'none'.  For cfg2 (SAVP,
64x64x3, 2 + 10 frames, B = 16) and the cfg3 shape (2 + 28 frames, B = 32), in alternating rounds: the median captured
training step and the median `generator_forward`, timed with CUDA events.  Then vp_lnorm_act and vp_lnorm_act_bwd alone
(next to vp_inorm_act / vp_inorm_act_bwd on the same tensor) at every norm extent of the cfg2 model: CUDA events around
back-to-back launches, GB/s from the algorithmic bytes (forward: read x, write y = 8 B per element, plus 8 B of stats per
sample; backward with one gradient source: read x and dy, write dx = 12 B per element, plus the stats and the gamma / beta
gradients) and that rate's share of the 3.35 TB/s HBM3 of an H100 SXM.  Prints the card's name, power limit and SM clocks
first, then one JSON line per row.
Usage: python tests/measure_norm_layer.py [--reps N] [--rounds R] [--configs cfg2,cfg3_shape] [--out FILE.json]"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from measure_conv_lstm import CONFIGS, L, card, time_model  # noqa: E402

NORMS = ('instance', 'layer', 'none')
HBM_BYTES_PER_S = 3.35e12
B_CFG2, S_CFG2 = 16, 11
# (positions, channels, act, samples per call) of the cfg2 model: generator h0..h5 and heads (NB = 2B), posterior encoder
# layers 2 and 3 (S * B samples, leaky relu)
EXTENTS = [(1024, 32, 'relu', 2 * B_CFG2), (256, 64, 'relu', 2 * B_CFG2), (64, 128, 'relu', 2 * B_CFG2),
           (4096, 32, 'relu', 2 * B_CFG2), (256, 128, 'lrelu', S_CFG2 * B_CFG2), (64, 256, 'lrelu', S_CFG2 * B_CFG2)]


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


def time_kernels(reps=200):
    rows = []
    for P, C, act_name, N in EXTENTS:
        act, alpha = (L.ACT_RELU, 0.0) if act_name == 'relu' else (L.ACT_LRELU, 0.2)
        gen = torch.Generator().manual_seed(P + C)
        x = torch.randn(N, P, C, generator=gen).cuda()
        dy = torch.randn(N, P, C, generator=gen).cuda()
        y, dx = torch.empty_like(x), torch.empty_like(x)
        g, b = torch.ones(C, device='cuda'), torch.zeros(C, device='cuda')
        dg, db = torch.zeros(C, device='cuda'), torch.zeros(C, device='cuda')
        lst, ist = torch.empty(N, 2, device='cuda'), torch.empty(N, C, 2, device='cuda')
        calls = {
            'lnorm_fwd': lambda: L.lnorm_act(x.data_ptr(), C, y.data_ptr(), C, N, P, C, g, b, act, alpha, lst),
            'lnorm_bwd': lambda: L.lnorm_act_bwd(x.data_ptr(), C, [(dy.data_ptr(), C)], dx.data_ptr(), C, N, P, C, g, b, lst, act, alpha,
                                                 dg, db),
            'inorm_fwd': lambda: L.inorm_act(x.data_ptr(), C, y.data_ptr(), C, N, P, C, g, b, act, alpha, ist),
            'inorm_bwd': lambda: L.inorm_act_bwd(x.data_ptr(), C, [(dy.data_ptr(), C)], dx.data_ptr(), C, N, P, C, g, b, ist, act, alpha,
                                                 dg, db),
        }
        calls['lnorm_fwd']()
        calls['inorm_fwd']()
        res = {}
        for rnd in range(3):                        # alternating
            for name, fn in calls.items():
                res.setdefault(name, []).append(_per_call_ms(fn, reps))
        elems = N * P * C
        nbytes = {'lnorm_fwd': 8 * elems + 8 * N, 'lnorm_bwd': 12 * elems + 8 * N + 8 * C}
        row = dict(extent='N=%d P=%d C=%d %s' % (N, P, C, act_name), mfloats=round(elems / 1e6, 3))
        for name, ts in res.items():
            t = sorted(ts)[1]
            row[name + '_us'] = round(t * 1000, 2)
            if name in nbytes:
                rate = nbytes[name] / (t * 1e-3)
                row[name + '_GBps'] = round(rate / 1e9, 1)
                row[name + '_hbm_share'] = round(rate / HBM_BYTES_PER_S, 3)
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None, help='also write every row to this JSON file')
    ap.add_argument('--configs', default=','.join(c[0] for c in CONFIGS), help='comma-separated subset of the configurations')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    for row in time_kernels():
        rows.append(row)
        print(json.dumps(row), flush=True)
    for name, hk, B in [c for c in CONFIGS if c[0] in args.configs.split(',')]:
        for rnd in range(args.rounds):
            for norm in NORMS:
                try:
                    step, fwd = time_model(dict(hk, norm_layer=norm), B, args.reps)
                except torch.cuda.OutOfMemoryError:
                    row = dict(config=name, B=B, norm_layer=norm, round=rnd, error='out of memory')
                    torch.cuda.empty_cache()
                else:
                    row = dict(config=name, B=B, norm_layer=norm, round=rnd, step_ms_median=round(step, 3),
                               generator_forward_ms_median=round(fwd, 3))
                rows.append(row)
                print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
