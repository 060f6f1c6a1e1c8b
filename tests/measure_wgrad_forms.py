"""Every form of the convolution weight gradient (vp_conv_wgrad) on every distinct wgrad call of the cfg2 training step.

The calls are recorded from one eager training step as in tests/measure_wgrad.py.  For each call this prints the form the
shape selects (lib.conv_wgrad_form: 32-row blocks per CTA x GEMM columns), its CTA count, SM fill (CTAs / (waves x SMs))
and 64-pixel stages per CTA, then the time of every form: a CUDA graph of `--inner` calls on fresh random operands,
replayed `--reps` times, median per call.  Each form's result on zeroed dW is also compared with the selected form's, bit
for bit.  The total lines give the step's time in the selected forms and in the fastest form of each call, and per form
the median over calls of time / (waves x stages per CTA).
Usage: python tests/measure_wgrad_forms.py [--reps N] [--inner N] [--out FILE.json]"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import measure_wgrad as M  # noqa: E402
from video_prediction_b200 import lib as L  # noqa: E402


def cdiv(a, b):
    return -(-a // b)


def time_form(run, reps, inner):
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(inner):
            run()
    graph.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        graph.replay()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / inner)
    del graph
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--inner', type=int, default=10)
    ap.add_argument('--out', default=None, help='also write every row to this JSON file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = [dict(card=M.card(), sms=sms)]
    print(json.dumps(rows[0]), flush=True)
    forms = L.conv_wgrad_forms()
    calls = M.record_step()
    counts = {}
    for c in calls:
        counts[c] = counts.get(c, 0) + 1
    lib = L.lib()
    picked_ms = best_ms = 0.0
    stage_cost = {f: [] for f in range(len(forms))}
    for key, cnt in sorted(counts.items(), key=lambda kv: str(kv[0])):
        xs, dys, geo, n_pad, kc, split_k = key
        g = L.VpConvGeom(*geo)
        form, ctas, splits, stages = L.conv_wgrad_form(g, xs[:5], dys[:5], n_pad, kc, sms, split_k)
        x, xv = M.view_of(xs, 1)
        dy, dyv = M.view_of(dys, 2)
        dw = torch.zeros(geo[0] * geo[1] * geo[2] * n_pad * kc * 32, device='cuda')
        shifted_c, plain_c = (dys[4], xs[4]) if geo[9] else (xs[4], dys[4])
        nblocks = geo[0] * geo[1] * geo[2] * cdiv(shifted_c, 32)
        ref = None
        per_form = {}
        for f, (blocks, bn) in enumerate(forms):
            run = lambda f=f: L.check(lib.vp_conv_wgrad_in_form(C.byref(xv), C.byref(dyv), C.byref(g), L.ptr(dw), n_pad, kc,
                                                                split_k, f, L.stream_ptr()))
            dw.zero_()
            run()
            out = dw.clone()
            ms = time_form(run, args.reps, args.inner)
            if f == form:
                ref = out
            waves = cdiv(cdiv(nblocks, blocks) * cdiv(plain_c, bn) * splits, sms)
            stage_cost[f].append(ms * 1e3 / (waves * stages))
            per_form['%dx%d' % (blocks, bn)] = (round(ms * 1e3, 1), out)
        same = {k: bool(torch.equal(v[1], ref)) for k, v in per_form.items()}
        times = {k: v[0] for k, v in per_form.items()}
        picked = times['%dx%d' % forms[form]]
        best = min(times.values())
        picked_ms += picked * cnt * 1e-3
        best_ms += best * cnt * 1e-3
        waves = cdiv(ctas, sms)
        row = dict(x=xs, dy=dys, geom=geo, n_pad=n_pad, kc=kc, calls_per_step=cnt, form='%dx%d' % forms[form], ctas=ctas,
                   sm_fill=round(ctas / (waves * sms), 3), splits=splits, stages_per_cta=stages, us_per_form=times,
                   picked_us=picked, best_us=best, same_bits_as_picked=all(same.values()))
        rows.append(row)
        print(json.dumps(row), flush=True)
        del x, dy, dw, ref, per_form
    costs = {'%dx%d' % forms[f]: round(statistics.median(v), 4) for f, v in stage_cost.items() if v}
    total = dict(total_calls=len(calls), distinct=len(counts), picked_ms_per_step=round(picked_ms, 3),
                 best_ms_per_step=round(best_ms, 3), median_stage_us=costs)
    rows.append(total)
    print(json.dumps(total), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
