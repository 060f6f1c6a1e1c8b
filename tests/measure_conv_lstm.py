"""Cost of the ConvLSTM's three forms: the instance-norm cell (the default), the norm-free cell (conv_rnn_norm_layer='none')
and its ablation (ablation_conv_rnn_norm: IN on the cell output).  For cfg2 (SAVP, 64x64x3, 2 + 10 frames, B = 16) and the
cfg3 shape (2 + 28 frames, B = 32), in alternating rounds: the median captured training step and the median
`generator_forward`, timed with CUDA events.  Then, per ConvLSTM layer of the cfg2 generator, vp_conv_lstm_fwd against the
same GEMM with the plain bias epilogue (vp_conv_igemm on the natural pack), CUDA events around back-to-back launches, with
TFLOP/s from the algorithmic FLOPs.  Prints the card's name, power limit and SM clocks first, then one JSON line per row.
Usage: python tests/measure_conv_lstm.py [--reps N] [--rounds R] [--configs cfg2,cfg3_shape] [--out FILE.json]"""
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
            video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, gan_feature_cdist_weight=0.0)
CONFIGS = [('cfg2', dict(SAVP, context_frames=2, sequence_length=12), 16),
           ('cfg3_shape', dict(SAVP, context_frames=2, sequence_length=30), 32)]
VARIANTS = [('instance', {}), ('none', dict(conv_rnn_norm_layer='none')), ('ablation', dict(ablation_conv_rnn_norm=True))]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def _events(fn, reps):
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def time_model(hk, B, reps, warmup=3):
    """Median captured training step and median generator_forward (ms)."""
    g = torch.Generator().manual_seed(0)
    model = get_model_class('savp')(mode='train', hparams_dict=hk)
    model.build_graph({'images': torch.rand(B, hk['sequence_length'], 64, 64, 3, generator=g)})
    model.use_cuda_graph = True
    for _ in range(warmup + 1):                     # step 0 runs eagerly; the graph is captured on the next one
        model.train_step()
    torch.cuda.synchronize()
    step = _events(model.train_step, reps)
    model.generator_forward()
    fwd = _events(model.generator_forward, reps)
    del model
    gc.collect()                                    # the layers refer back to the model: free its buffers before the next one
    torch.cuda.empty_cache()
    return step, fwd


def time_layers(B, reps=50):
    """Each ConvLSTM gate convolution of the cfg2 generator (NB = 2B) with the cell epilogue and with the bias epilogue."""
    rows = []
    nb = 2 * B
    for hw, F in ((32, 32), (16, 64), (8, 128)):
        ci = 2 * F + 8
        gen = torch.Generator().manual_seed(F)
        x = torch.randn(nb, hw, hw, ci, generator=gen).cuda()
        w = (torch.randn(5, 5, ci, 4 * F, generator=gen) * 0.03).cuda()
        bias = torch.zeros(4 * F, device='cuda')
        c_prev = torch.randn(nb, hw, hw, F, generator=gen).cuda()
        c_new, z, h = (torch.empty(nb, hw, hw, n, device='cuda') for n in (F, 4 * F, F))
        nat, n_pad, kc = L.pack_weights(w, (1, 5, 5), ci, 4 * F, L.WKIND_PLAIN, L.WLAYOUT_FWD)
        gat, _, _ = L.pack_weights(w, (1, 5, 5), ci, 4 * F, L.WKIND_PLAIN, L.WLAYOUT_FWD | L.WLAYOUT_GATES)
        g = L.geom((1, 5, 5), (1, 1, 1), (0, 2, 2))
        xv, zv = L.tensor_view(x, ci), L.tensor_view(z)
        dests = [(h.data_ptr(), F)]
        calls = {'bias_epilogue': lambda: L.conv_igemm(xv, g, nat, n_pad, kc, zv, bias),
                 'lstm_epilogue': lambda: L.conv_lstm_fwd(xv, g, gat, n_pad, kc, z, bias, c_prev, c_new, dests)}
        flops = 2.0 * nb * hw * hw * 4 * F * ci * 25
        res = {}
        for rnd in range(3):                        # alternating
            for name, fn in calls.items():
                fn()
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(reps):
                    fn()
                b.record()
                b.synchronize()
                res.setdefault(name, []).append(a.elapsed_time(b) / reps)
        row = dict(layer='%dx%d F=%d ci=%d NB=%d' % (hw, hw, F, ci, nb), gflop=round(flops / 1e9, 3))
        for name, ts in res.items():
            t = sorted(ts)[1]
            row[name + '_us'] = round(t * 1000, 2)
            row[name + '_tflops'] = round(flops / (t * 1e-3) / 1e12, 1)
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
    for name, hk, B in [c for c in CONFIGS if c[0] in args.configs.split(',')]:
        for rnd in range(args.rounds):
            for vname, v in VARIANTS:
                try:
                    step, fwd = time_model(dict(hk, **v), B, args.reps)
                except torch.cuda.OutOfMemoryError:
                    row = dict(config=name, B=B, variant=vname, round=rnd, error='out of memory')
                    gc.collect()
                    torch.cuda.empty_cache()
                else:
                    row = dict(config=name, B=B, variant=vname, round=rnd, step_ms_median=round(step, 3),
                               generator_forward_ms_median=round(fwd, 3))
                rows.append(row)
                print(json.dumps(row), flush=True)
    for row in time_layers(16):
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
