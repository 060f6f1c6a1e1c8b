"""Cost of the per-frame image discriminator over the sampled clip (`images_sn_gan_weight`, `images_sn_vae_gan_weight`).
cfg2 (SAVP, 64x64x3, 2 + 10 frames, B = 16) with and without both images weights at 0.1, in alternating rounds: the median
captured training step, timed with CUDA events.  Then, per layer of the `discriminator/images` tower (N = 2 B clip = 320
frames) and, for comparison, of the `discriminator/video` tower (32 clips of 10 frames), the launches the step makes -- the
forward (leaky relu epilogue), the input gradient with the fused leaky-relu gradient, and the weight gradient with its
spectral-norm backward -- CUDA events around back-to-back launches, with TFLOP/s from the algorithmic FLOPs.  Prints the
card's name, power limit and SM clocks first, then one JSON line per row.
Usage: python tests/measure_images_discriminator.py [--reps N] [--rounds R] [--out FILE.json]"""
import argparse
import gc
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from video_prediction_b200.models import get_model_class  # noqa: E402

CFG2 = dict(lr=0.0002, beta1=0.5, beta2=0.999, l1_weight=100.0, l2_weight=0.0, kl_weight=1.0, video_sn_vae_gan_weight=0.1,
            video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, gan_feature_cdist_weight=0.0, context_frames=2,
            sequence_length=12)
IMAGES = dict(images_sn_gan_weight=0.1, images_sn_vae_gan_weight=0.1)
B = 16


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


def _model(hk):
    g = torch.Generator().manual_seed(0)
    model = get_model_class('savp')(mode='train', hparams_dict=hk)
    model.build_graph({'images': torch.rand(B, hk['sequence_length'], 64, 64, 3, generator=g)})
    return model


def _free(model):
    del model
    gc.collect()                                    # the layers refer back to the model: free its buffers before the next one
    torch.cuda.empty_cache()


def time_step(hk, reps, warmup=3):
    """Median captured training step (ms)."""
    model = _model(hk)
    model.use_cuda_graph = True
    for _ in range(warmup + 1):                     # step 0 runs eagerly; the graph is captured on the next one
        model.train_step()
    torch.cuda.synchronize()
    t = _events(model.train_step, reps)
    _free(model)
    return t


def _launch_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def time_layers(reps):
    """Each layer of the images and the video tower of the root scope on a full 2B batch, after one training step."""
    model = _model(dict(CFG2, **IMAGES))
    model.train_step()
    torch.cuda.synchronize()
    rows = []
    for scope in ('discriminator/images', 'discriminator/video'):
        net = model.dnets[scope]
        model._d_sn_and_pack(net)
        nb = net['clip'].shape[0]
        for l, lay in enumerate(net['layers']):
            x = net['clip'] if l == 0 else net['feat'][l - 1]
            y, dy = net['feat'][l], net['dfeat'][l]
            dy.copy_(torch.randn_like(dy) * 1e-3)
            dx = net['dclip'] if l == 0 else net['dfeat'][l - 1]
            act_y = None if l == 0 else x
            out_pos = int(np.prod(y.shape[:-1]))
            flops = 2.0 * out_pos * lay.co * int(np.prod(lay.k3)) * lay.cin_ref
            calls = {'fwd': lambda: lay.fwd(x, y), 'dgrad': lambda: lay.dgrad(dy, dx, act_y=act_y), 'wgrad_sn': lambda: lay.wgrad(x, dy)}
            res = {}
            for _ in range(3):                      # alternating rounds, the middle one kept
                for name, fn in calls.items():
                    res.setdefault(name, []).append(_launch_time(fn, reps))
            row = dict(tower=scope.split('/')[-1], layer=lay.wname.split('/')[-3], frames=nb * x.shape[1], input=list(x.shape[1:]),
                       co=lay.co, gflop=round(flops / 1e9, 3))
            for name, ts in res.items():
                t = sorted(ts)[1]
                row[name + '_us'] = round(t * 1000, 2)
                row[name + '_tflops'] = round(flops / (t * 1e-3) / 1e12, 1)
            rows.append(row)
    _free(model)
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
    for rnd in range(args.rounds):
        for vname, hk in (('cfg2', CFG2), ('cfg2+images', dict(CFG2, **IMAGES))):
            row = dict(config=vname, B=B, round=rnd, step_ms_median=round(time_step(hk, args.reps), 3))
            rows.append(row)
            print(json.dumps(row), flush=True)
    for row in time_layers(args.reps):
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
