"""Timing ablation of the cfg2 training step: the step is re-captured with one kernel family not launched (VP_SKIP, results
are wrong by design) and the difference to the full step is that family's REAL cost inside the CUDA graph (warm L2, overlap
with the parallel branches), which per-launch timings (cold caches, serialised) do not show."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
fams = (sys.argv[1].split(';') if len(sys.argv) > 1 else ['', 'inorm', 'gates', 'wgrad', 'c4wgrad', 'pack', 'colsum,copy', 'cdna', 'sn', 'cosd,dense', 'adam'])
base = None
for f in fams:
    env = dict(os.environ, VP_SKIP=f)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--steps', '10', '--warmup', '3', '--no-cpu', '--no-roofline'], env=env,
                       capture_output=True, text=True)
    line = [l for l in r.stdout.splitlines() if l.startswith('{')]
    if not line:
        print('%-14s FAILED %s' % (f, r.stderr[-300:]))
        continue
    ms = json.loads(line[-1])['ms_per_step']
    if base is None:
        base = ms
    print('skip %-14s %7.2f ms/step   (family cost %.2f ms = %.1f %%)' % (f or '-', ms, base - ms, 100 * (base - ms) / base))
    sys.stdout.flush()
