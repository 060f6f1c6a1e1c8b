"""Per-call cost of the engine's forward / dgrad kernel in the cfg2 training step, with the tile form each call runs.

Records and times the calls exactly as tests/measure_engine_fwd.py does (one eager cfg2 step records them; each distinct
call is replayed on fresh operands in a CUDA graph of `--inner` calls, median over `--reps` replays).  The form (pixel
rows x GEMM columns of a tile) is the one conv_igemm_impl picks, read from the library (lib.conv_igemm_form); the grid
follows from it by the launch code: m-tiles, n-tiles, CTAs launched, the share of the SMs they occupy and the pixel
tiles each CTA walks.  Prints the card first, then one JSON line per distinct call, sorted by time per step, then a total.
Usage: python tests/measure_engine_forms.py [--root DIR] [--reps N] [--inner N] [--out FILE.json]"""
import argparse
import json
import os
import sys

import torch

import measure_engine_fwd as M


def grid(L, key, sms):
    """(rows, BN, m-tiles, n-tiles, CTAs, tiles per CTA) of the call."""
    kind, xs, geo, n_pad, kc, os_, _, _, split_k, _ = key
    kd, kh, kw, sd, sh, sw, pd, ph, pw, tr = geo
    if kind == 'lstm':
        lat, (rows, bn) = [os_[2], os_[1], 1, os_[0]], (128, 128)
    else:
        lat = [os_[3], os_[2], os_[1], os_[0]]
        rows, bn = L.conv_igemm_form(L.VpConvGeom(*geo), os_[:4], n_pad, kc, sms, split_k)
    phases = sd * sh * sw if tr else 1
    if tr:
        lat = [-(-lat[0] // sw), -(-lat[1] // sh), -(-lat[2] // sd), lat[3]]
    rem, m_tiles = rows, 1
    for e in lat[:3]:
        b = min(1 << (max(e, 1).bit_length() - 1), rem)
        rem //= b
        m_tiles *= -(-e // b)
    m_tiles *= -(-lat[3] // rem)
    n_tiles = -(-n_pad // bn)
    other = n_tiles * phases * max(1, split_k)
    gx = min(m_tiles, max(1, sms // other))
    return rows, bn, m_tiles, n_tiles, gx * other, -(-m_tiles // gx)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--root', default=M.HERE, help='tree to import video_prediction_b200 (and bench.py) from')
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--inner', type=int, default=20)
    ap.add_argument('--out', default=None, help='also write every row to this JSON file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    sys.path.insert(0, os.path.abspath(args.root))
    import bench
    from video_prediction_b200 import lib as L
    print(json.dumps(dict(card=M.card(), root=os.path.abspath(args.root))), flush=True)
    counts = {}
    for c in M.record_step(L, bench):
        counts[c] = counts.get(c, 0) + 1
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = []
    for key, cnt in counts.items():
        ms, flops = M.time_call(L, key, args.reps, args.inner)
        r, bn, m_tiles, n_tiles, ctas, per_cta = grid(L, key, sms)
        rows.append(dict(kind=key[0], x=key[1], geom=key[2], n_pad=key[3], kc=key[4], out=key[5], rows=r, bn=bn,
                         m_tiles=m_tiles, n_tiles=n_tiles, ctas=ctas, sm_fill=round(min(ctas, sms) / sms, 3),
                         tiles_per_cta=per_cta, calls_per_step=cnt, us_per_call=round(ms * 1e3, 2),
                         tflops=round(flops / ms * 1e-9, 2), ms_per_step=round(ms * cnt, 3), flops=flops * cnt))
    rows.sort(key=lambda r: -r['ms_per_step'])
    for r in rows:
        print(json.dumps({k: v for k, v in r.items() if k != 'flops'}), flush=True)
    tot_ms, tot_flops = sum(r['ms_per_step'] for r in rows), sum(r.pop('flops') for r in rows)
    total = dict(total_calls=sum(counts.values()), distinct=len(rows), ms_per_step=round(tot_ms, 3),
                 tflop_per_step=round(tot_flops * 1e-12, 3), tflops=round(tot_flops / tot_ms * 1e-9, 2))
    print(json.dumps(total), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows + [total], f, indent=1)


if __name__ == '__main__':
    main()
