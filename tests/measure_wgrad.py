"""Per-layer cost of the convolution weight gradient (vp_conv_wgrad) in the cfg2 training step (SAVP, B = 16).

The calls and their shapes are read from a built model: one eager training step runs with lib.conv_wgrad recording its
arguments.  Each distinct call (geometry, operand extents and channel counts) is then replayed on fresh random operands of
the same shape with split_k = 0, as the model calls it, and timed with CUDA events around `--inner` back-to-back calls after
warm-up; the median over `--reps` such windows is reported.  Prints the card name, power limit and SM clock first, then one
JSON line per distinct call (time, algorithmic TFLOP/s counted as lib.conv_wgrad counts them, operand bytes read, calls per
step) and a total line.  Usage: python tests/measure_wgrad.py [--reps N] [--inner N] [--out FILE.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench  # noqa: E402
from video_prediction_b200 import lib as L  # noqa: E402
from video_prediction_b200.models import get_model_class  # noqa: E402

HPARAMS = bench.CONFIGS['cfg2']['hparams']
B = bench.CONFIGS['cfg2']['batch']


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def record_step():
    """Runs one eager training step of cfg2 and returns the argument tuples of every lib.conv_wgrad call in it."""
    g = torch.Generator().manual_seed(0)
    inp = {'images': torch.rand(B, HPARAMS['sequence_length'], 64, 64, 3, generator=g)}
    model = get_model_class('savp')(mode='train', hparams_dict=dict(HPARAMS), num_gpus=1)
    model.build_graph(inp)
    model.use_cuda_graph = False
    calls = []
    real = L.conv_wgrad

    def spy(x_view, dy_view, g, dwpacked, n_pad, kc, split_k=1):
        t = lambda v: (v.n, v.d, v.h, v.w, v.c, v.cstride)
        geo = (g.kd, g.kh, g.kw, g.sd, g.sh, g.sw, g.pd, g.ph, g.pw, g.transposed)
        calls.append((t(x_view), t(dy_view), geo, n_pad, kc, split_k))
        return real(x_view, dy_view, g, dwpacked, n_pad, kc, split_k)

    L.conv_wgrad = spy
    try:
        model.train_step(inp)
        torch.cuda.synchronize()
    finally:
        L.conv_wgrad = real
    del model
    torch.cuda.empty_cache()
    return calls


def view_of(shape, seed):
    n, d, h, w, c, cs = shape
    gen = torch.Generator().manual_seed(seed)
    t = torch.randn(n, d, h, w, cs, generator=gen).cuda()
    return t, L.VpTensor(t.data_ptr(), n, d, h, w, c, cs)


def time_call(key, reps, inner):
    xs, dys, geo, n_pad, kc, split_k = key
    x, xv = view_of(xs, 1)
    dy, dyv = view_of(dys, 2)
    g = L.VpConvGeom(*geo)
    dw = torch.zeros(geo[0] * geo[1] * geo[2] * n_pad * kc * 32, device='cuda')
    lib = L.lib()
    run = lambda: L.check(lib.vp_conv_wgrad(C.byref(xv), C.byref(dyv), C.byref(g), L.ptr(dw), n_pad, kc, split_k, L.stream_ptr()))
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(inner):
            run()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / inner)
    times.sort()
    del x, dy, dw
    taps = geo[0] * geo[1] * geo[2] / (float(geo[3] * geo[4] * geo[5]) if geo[9] else 1.0)
    flops = 2.0 * dys[0] * dys[1] * dys[2] * dys[3] * dys[4] * xs[4] * taps
    nbytes = 4 * (xs[0] * xs[1] * xs[2] * xs[3] * xs[4] + dys[0] * dys[1] * dys[2] * dys[3] * dys[4])
    return times[len(times) // 2], flops, nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--inner', type=int, default=10)
    ap.add_argument('--out', default=None, help='also write every row to this JSON file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    calls = record_step()
    counts = {}
    for c in calls:
        counts[c] = counts.get(c, 0) + 1
    tot_ms = tot_flops = tot_bytes = 0.0
    for key, cnt in sorted(counts.items(), key=lambda kv: str(kv[0])):
        ms, flops, nbytes = time_call(key, args.reps, args.inner)
        row = dict(x=key[0], dy=key[1], geom=key[2], n_pad=key[3], kc=key[4], split_k=key[5], calls_per_step=cnt,
                   ms_per_call=round(ms, 4), tflops=round(flops / ms * 1e-9, 2), bytes_read=nbytes,
                   ms_per_step=round(ms * cnt, 3))
        tot_ms += ms * cnt
        tot_flops += flops * cnt
        tot_bytes += nbytes * cnt
        rows.append(row)
        print(json.dumps(row), flush=True)
    total = dict(total_calls=len(calls), distinct=len(counts), ms_per_step=round(tot_ms, 3),
                 tflop_per_step=round(tot_flops * 1e-12, 3), tflops=round(tot_flops / tot_ms * 1e-9, 2),
                 gb_read_per_step=round(tot_bytes * 1e-9, 3))
    rows.append(total)
    print(json.dumps(total), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
