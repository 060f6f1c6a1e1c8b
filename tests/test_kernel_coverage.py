"""Every C entry point of the CUDA library has a direct GPU test (runs without a GPU).

The entry points are the `extern "C"` vp_* functions of video_prediction_b200/csrc/*.cu.  Each is reached from Python
through the top-level function or class of lib.py whose body calls `lib().vp_X(`.  Some tests/test_gpu_*.py must call
the entry point itself (`vp_X(`) or that wrapper (`L.wrapper(` / `lib.wrapper(`); being reached only through a whole
training step does not count.  Only the three bookkeeping functions of api.cu have no test of their own."""
import ast
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'video_prediction_b200')
ALLOWED = {'vp_last_error', 'vp_launch_count', 'vp_version'}


def entry_points():
    names = set()
    for path in glob.glob(os.path.join(PKG, 'csrc', '*.cu')):
        with open(path) as f:
            names.update(re.findall(r'extern\s+"C"\s+[\w\s\*]*?\b(vp_\w+)\s*\(', f.read()))
    return names


def wrappers():
    """vp_X -> names of the top-level lib.py functions / classes that call lib().vp_X(."""
    with open(os.path.join(PKG, 'lib.py')) as f:
        src = f.read()
    out = {}
    for node in ast.parse(src).body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)):
            for ep in re.findall(r'\blib\(\)\.(vp_\w+)\(', ast.get_source_segment(src, node)):
                out.setdefault(ep, set()).add(node.name)
    return out


def untested(test_sources):
    wr = wrappers()
    missing = []
    for ep in sorted(entry_points() - ALLOWED):
        pats = [r'\b%s\(' % ep] + [r'\b(?:L|lib)\.%s\(' % w for w in sorted(wr.get(ep, ()))]
        if not any(re.search(p, s) for p in pats for s in test_sources):
            missing.append((ep, sorted(wr.get(ep, ()))))
    return missing


def _gpu_test_sources():
    out = []
    for path in sorted(glob.glob(os.path.join(ROOT, 'tests', 'test_gpu_*.py'))):
        with open(path) as f:
            out.append(f.read())
    return out


def test_the_parser_finds_the_library():
    eps, wr = entry_points(), wrappers()
    assert len(eps) > 60 and ALLOWED <= eps
    assert {'vp_conv_igemm', 'vp_gan_loss', 'vp_spectral_norm_bwd', 'vp_adam'} <= eps
    assert wr['vp_pack_weights_batch'] == {'PackPlan'}
    assert wr['vp_cdna_slots_bwd'] == {'slots_bwd'} and wr['vp_flow_slots_bwd'] == {'slots_bwd'}
    assert wr['vp_gan_loss'] == {'gan_loss'}


def test_every_entry_point_has_a_gpu_test():
    missing = untested(_gpu_test_sources())
    assert not missing, 'C entry points (and their lib.py wrappers) no tests/test_gpu_*.py calls: %s' % missing


def test_the_guard_notices_a_missing_test():
    """Without the file that holds its only direct test, an entry point is reported."""
    sources = [s for s in _gpu_test_sources() if 'L.kl_loss(' not in s]
    assert ('vp_kl_loss', ['kl_loss']) in untested(sources)
