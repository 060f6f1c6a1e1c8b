"""Per-call cost of the engine's forward / dgrad kernel (vp_conv_igemm, vp_conv_igemm_actgrad, vp_conv_lstm_fwd) in the cfg2
training step (SAVP, B = 16).

The calls and their shapes are read from a built model: one eager training step runs with lib.conv_igemm,
lib.conv_igemm_actgrad and lib.conv_lstm_fwd recording their arguments.  Each distinct call is then replayed on fresh
random operands of the same shape: `--inner` back-to-back calls are captured in a CUDA graph, the graph is replayed between
CUDA events, and the median over `--reps` replays is reported.  Prints the card name, power limit and SM clock first, then
one JSON line per distinct call (geometry, the kernel's launch shape as igemm.cu derives it, time, algorithmic TFLOP/s
counted as lib.py counts them, calls per step) and a total line.  `--root DIR` imports video_prediction_b200 from the tree
DIR (built there), so that two trees can be timed in one process each on the same card.
Usage: python tests/measure_engine_fwd.py [--root DIR] [--reps N] [--inner N] [--out FILE.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def vshape(v):
    return (v.n, v.d, v.h, v.w, v.c, v.cstride)


def gshape(g):
    return (g.kd, g.kh, g.kw, g.sd, g.sh, g.sw, g.pd, g.ph, g.pw, g.transposed)


def record_step(L, bench):
    """Runs one eager training step of cfg2 and returns one key per engine forward / dgrad call in it."""
    from video_prediction_b200.models import get_model_class
    hp, B = bench.CONFIGS['cfg2']['hparams'], bench.CONFIGS['cfg2']['batch']
    g = torch.Generator().manual_seed(0)
    inp = {'images': torch.rand(B, hp['sequence_length'], 64, 64, 3, generator=g)}
    model = get_model_class('savp')(mode='train', hparams_dict=dict(hp), num_gpus=1)
    model.build_graph(inp)
    model.use_cuda_graph = False
    calls = []
    real = L.conv_igemm, L.conv_igemm_actgrad, L.conv_lstm_fwd

    def igemm(x_view, g, wpacked, n_pad, kc, out_view, bias=None, act=L.ACT_NONE, alpha=0.0, split_k=1, accumulate=0):
        calls.append(('igemm', vshape(x_view), gshape(g), n_pad, kc, vshape(out_view), bias is not None, act, split_k,
                      accumulate))
        return real[0](x_view, g, wpacked, n_pad, kc, out_view, bias, act, alpha, split_k, accumulate)

    def actgrad(x_view, g, wpacked, n_pad, kc, out_view, act_output_addr, addend_addr, act, alpha=0.0, accumulate=0):
        calls.append(('actgrad', vshape(x_view), gshape(g), n_pad, kc, vshape(out_view), bool(addend_addr), act, 1,
                      accumulate))
        return real[1](x_view, g, wpacked, n_pad, kc, out_view, act_output_addr, addend_addr, act, alpha, accumulate)

    def lstm(x_view, g, wpacked, n_pad, kc, z, bias, c_prev, c_new, h_dsts, accumulate=0, forget_bias=1.0):
        zs = tuple(z.shape)
        calls.append(('lstm', vshape(x_view), gshape(g), n_pad, kc, (zs[0] * (zs[1] if len(zs) == 5 else 1),) + zs[-3:],
                      tuple(cs for _, cs in h_dsts), 0, 1, accumulate))
        return real[2](x_view, g, wpacked, n_pad, kc, z, bias, c_prev, c_new, h_dsts, accumulate, forget_bias)

    L.conv_igemm, L.conv_igemm_actgrad, L.conv_lstm_fwd = igemm, actgrad, lstm
    try:
        model.train_step(inp)
        torch.cuda.synchronize()
    finally:
        L.conv_igemm, L.conv_igemm_actgrad, L.conv_lstm_fwd = real
    del model
    torch.cuda.empty_cache()
    return calls


def launch_shape(key, sms):
    """(BN, m-tiles, n-tiles, tiles per CTA, k-chunks per tile) of the call, by the rules of conv_igemm_impl."""
    kind, xs, geo, n_pad, kc, os_, _, _, split_k, _ = key
    kd, kh, kw, sd, sh, sw, pd, ph, pw, tr = geo
    if kind == 'lstm':
        lat = [os_[2], os_[1], 1, os_[0]]
    else:
        lat = [os_[3], os_[2], os_[1], os_[0]]
    if tr:
        lat = [-(-lat[0] // sw), -(-lat[1] // sh), -(-lat[2] // sd), lat[3]]
        phase_taps = [len(range((f + p) % s, k, s)) for f, p, s, k in ((0, pd, sd, kd), (0, ph, sh, kh), (0, pw, sw, kw))]
        phases, taps = sd * sh * sw, max(1, phase_taps[0] * phase_taps[1] * phase_taps[2])
    else:
        phases, taps = 1, kd * kh * kw
    rem, box = 128, []
    for e in lat[:3]:
        b = min(1 << (max(e, 1).bit_length() - 1), rem)
        box.append(b)
        rem //= b
    box.append(rem)
    m_tiles = 1
    for e, b in zip(lat, box):
        m_tiles *= -(-e // b)
    bn = 128 if kind == 'lstm' else min((128, 64, 32), key=lambda b: (-(-n_pad // b) * b, -b))
    n_tiles = -(-n_pad // bn)
    splits = max(1, min(split_k if split_k > 0 else 1, taps * kc))
    gx = min(m_tiles, max(1, sms // (n_tiles * phases * splits)))
    return bn, m_tiles, n_tiles, -(-m_tiles // gx), taps * kc // splits


def rnd(numel, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(numel, generator=g).cuda()


def time_call(L, key, reps, inner):
    kind, xs, geo, n_pad, kc, os_, flag, act, split_k, accumulate = key
    x = rnd(xs[0] * xs[1] * xs[2] * xs[3] * xs[5], 1)
    xv = L.VpTensor(x.data_ptr(), *xs)
    g = L.VpConvGeom(*geo)
    w = rnd(geo[0] * geo[1] * geo[2] * n_pad * kc * 32, 2) * 0.05
    keep = [x, w]
    if kind == 'lstm':
        pix = os_[0] * os_[1] * os_[2]
        f = os_[3] // 4
        z = torch.zeros(os_, device='cuda')
        bias, c_prev, c_new = rnd(4 * f, 3), rnd(pix * f, 4), torch.zeros(pix * f, device='cuda')
        hs = [torch.zeros(pix * cs, device='cuda') for cs in flag]
        keep += [z, bias, c_prev, c_new] + hs
        zv = L.tensor_view(z)
        pa = (C.c_void_p * len(hs))(*[C.c_void_p(h.data_ptr()) for h in hs])
        sa = (C.c_int * len(hs))(*flag)
        run = lambda: L.check(L.lib().vp_conv_lstm_fwd(C.byref(xv), C.byref(g), L.ptr(w), n_pad, kc, C.byref(zv), L.ptr(bias),
                                                        L.ptr(c_prev), L.ptr(c_new), pa, sa, len(hs), C.c_float(1.0),
                                                        accumulate, L.stream_ptr()))
        flops = 2.0 * pix * os_[3] * xs[4] * geo[0] * geo[1] * geo[2]
    else:
        out = rnd(os_[0] * os_[1] * os_[2] * os_[3] * os_[5], 3)
        ov = L.VpTensor(out.data_ptr(), *os_)
        keep.append(out)
        if kind == 'actgrad':
            y = torch.sigmoid(rnd(out.numel(), 4))
            add = rnd(out.numel(), 5) if flag else None
            keep += [y, add]
            run = lambda: L.check(L.lib().vp_conv_igemm_actgrad(C.byref(xv), C.byref(g), L.ptr(w), n_pad, kc, C.byref(ov),
                                                                C.c_void_p(y.data_ptr()), L.ptr(add), act, C.c_float(0.2),
                                                                accumulate, L.stream_ptr()))
        else:
            bias = rnd(n_pad, 6) if flag else None
            keep.append(bias)
            run = lambda: L.check(L.lib().vp_conv_igemm(C.byref(xv), C.byref(g), L.ptr(w), n_pad, kc, C.byref(ov), L.ptr(bias),
                                                        act, C.c_float(0.2), split_k, accumulate, L.stream_ptr()))
        taps = geo[0] * geo[1] * geo[2] / (float(geo[3] * geo[4] * geo[5]) if geo[9] else 1.0)
        flops = 2.0 * os_[0] * os_[1] * os_[2] * os_[3] * os_[4] * xs[4] * taps
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
    times.sort()
    del graph, keep
    return times[len(times) // 2], flops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--root', default=HERE, help='tree to import video_prediction_b200 (and bench.py) from')
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--inner', type=int, default=20)
    ap.add_argument('--out', default=None, help='also write every row to this JSON file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    sys.path.insert(0, os.path.abspath(args.root))
    import bench
    from video_prediction_b200 import lib as L
    rows = [dict(card=card(), root=os.path.abspath(args.root))]
    print(json.dumps(rows[0]), flush=True)
    calls = record_step(L, bench)
    counts = {}
    for c in calls:
        counts[c] = counts.get(c, 0) + 1
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tot_ms = tot_flops = 0.0
    for key, cnt in sorted(counts.items(), key=lambda kv: str(kv[0])):
        ms, flops = time_call(L, key, args.reps, args.inner)
        bn, m_tiles, n_tiles, per_cta, chunks = launch_shape(key, sms)
        row = dict(kind=key[0], x=key[1], geom=key[2], n_pad=key[3], kc=key[4], out=key[5], act=key[7], accumulate=key[9],
                   bn=bn, m_tiles=m_tiles, n_tiles=n_tiles, tiles_per_cta=per_cta, kchunks_per_tile=chunks,
                   calls_per_step=cnt, us_per_call=round(ms * 1e3, 2), tflops=round(flops / ms * 1e-9, 2),
                   ms_per_step=round(ms * cnt, 3))
        tot_ms += ms * cnt
        tot_flops += flops * cnt
        rows.append(row)
        print(json.dumps(row), flush=True)
    total = dict(total_calls=len(calls), distinct=len(counts), ms_per_step=round(tot_ms, 3),
                 tflop_per_step=round(tot_flops * 1e-12, 3), tflops=round(tot_flops / tot_ms * 1e-9, 2))
    rows.append(total)
    print(json.dumps(total), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
