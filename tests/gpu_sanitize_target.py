"""Small invocations of every hand-written tensor-core / cluster kernel for compute-sanitizer (memcheck / racecheck):
   compute-sanitizer --tool memcheck python tests/gpu_sanitize_target.py
Sizes are tiny so that the instrumented run takes seconds; results are still checked against fp64 references, and the
reductions that replace float atomics (engine weight-gradient splits, first-layer weight gradient) are run twice and must
agree bit for bit."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.nn.functional as F
from video_prediction_b200 import lib as L


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).cuda()


def as5(t):
    """[N, H, W, C] -> [N, 1, H, W, C]; [N, D, H, W, C] unchanged."""
    return t.unsqueeze(1) if t.dim() == 4 else t


def ref_conv(x, w, s, p):
    """fp64 conv3d of channels-last x with DHWIO weights w (kd, kh, kw, ci, co) -> channels-last [N, D, H, W, co]."""
    y = F.conv3d(as5(x).double().permute(0, 4, 1, 2, 3), w.double().permute(4, 3, 0, 1, 2), stride=s, padding=p)
    return y.permute(0, 2, 3, 4, 1)


ok = True
# forward engine (wgmma): 2-D stride 1 (gate conv), 2-D stride 2, 3-D stride 1, 3-D stride (1,2,2); N tiles 128 / 64 / 32
for name, xs, cin, cout, k, s, p in (('gate 5x5', (2, 16, 16), 72, 128, (1, 5, 5), (1, 1, 1), (0, 2, 2)),
                                     ('4x4 s2', (2, 16, 16), 40, 64, (1, 4, 4), (1, 2, 2), (0, 1, 1)),
                                     ('conv3d k3', (2, 4, 16, 16), 32, 32, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
                                     ('conv3d k4 s(1,2,2)', (2, 5, 16, 16), 32, 64, (4, 4, 4), (1, 2, 2), (1, 1, 1))):
    x = rnd(*xs, cin)
    w = rnd(*k, cin, cout, seed=1, scale=0.05)
    ref = ref_conv(x, w, s, p)
    oshape = tuple(ref.shape[:-1]) if len(xs) == 4 else (ref.shape[0],) + tuple(ref.shape[2:-1])
    wp, n_pad, kc = L.pack_weights(w if len(xs) == 4 else w[0], k, cin, cout, L.WKIND_PLAIN, L.WLAYOUT_FWD, ci_int=cin)
    out = torch.zeros(*oshape, cout, device='cuda')
    L.conv_igemm(L.tensor_view(x, cin), L.geom(k, s, p, False), wp, n_pad, kc, L.tensor_view(out, cout), None, 0, 0.0, 0)
    torch.cuda.synchronize()
    err = (as5(out).double() - ref).abs().max().item() / (ref.abs().max().item() + 1e-30)
    print('%-22s forward rel err vs fp64 %.1e' % (name, err))
    ok &= err < 3e-3
# weight gradients (mma.sync, pixel-range splits reduced in order): against the fp64 autograd gradient, twice bit-identical
for name, xs, cin, cout, k, s, p in (('wgrad 5x5', (4, 16, 16), 72, 128, (1, 5, 5), (1, 1, 1), (0, 2, 2)),
                                     ('wgrad k4 s(1,2,2)', (2, 5, 16, 16), 32, 64, (4, 4, 4), (1, 2, 2), (1, 1, 1))):
    x = rnd(*xs, cin)
    w = rnd(*k, cin, cout, seed=1, scale=0.05).double().requires_grad_()
    ref_y = ref_conv(x, w, s, p)
    dy5 = rnd(*ref_y.shape, seed=2)
    ref_y.backward(dy5.double())
    dy = (dy5[:, 0] if len(xs) == 3 else dy5).contiguous()          # 2-D inputs have no depth axis
    n_pad, kc = L.pad_to(cout, 16), L.pad_to(cin, 32) // 32
    taps = k[0] * k[1] * k[2]
    runs = []
    for _ in range(2):
        dwp = torch.zeros(taps * n_pad * kc * 32, device='cuda')
        L.conv_wgrad(L.tensor_view(x, cin), L.tensor_view(dy, cout), L.geom(k, s, p, False), dwp, n_pad, kc, 0)
        runs.append(dwp)
    torch.cuda.synchronize()
    got = runs[0].view(taps, n_pad, kc * 32)[:, :cout, :cin].double()                 # [tap][co][ci]
    ref = w.grad.reshape(taps, cin, cout).transpose(1, 2)
    err = ((got - ref).norm() / ref.norm()).item()
    same = bool(torch.equal(runs[0], runs[1]))
    print('%-22s rel L2 err vs fp64 %.1e, two runs bit-identical %s' % (name, err, same))
    ok &= err < 3e-3 and same
# slab / cluster plane kernels
N, P, C = 4, 1024, 32
x, g, b = rnd(N, P, C) + 2.0, rnd(C, seed=1) * 0.3 + 1, rnd(C, seed=2)
y, st = torch.zeros(N, P, C, device='cuda'), torch.zeros(N, C, 2, device='cuda')
L.inorm_act(x.data_ptr(), C, y.data_ptr(), C, N, P, C, g, b, L.ACT_RELU, 0.0, st)
xd = x.double()
ref = torch.relu((xd - xd.mean(1, keepdim=True)) * torch.rsqrt(xd.var(1, unbiased=False, keepdim=True) + 1e-6) * g.double() + b.double())
err = (y.double() - ref).abs().max().item()
print('slab instance norm (cluster of %d): max err %.1e' % (8, err))
ok &= err < 1e-4
Fl = 32
pre, c0 = rnd(N, P, 4 * Fl), rnd(N, P, Fl, seed=3)
g1, b1, g2, b2 = torch.ones(4 * Fl, device='cuda'), torch.zeros(4 * Fl, device='cuda'), torch.ones(Fl, device='cuda'), torch.zeros(Fl, device='cuda')
c1, h = torch.zeros(N, P, Fl, device='cuda'), torch.zeros(N, P, Fl, device='cuda')
s1, s2 = torch.zeros(N, 4 * Fl, 2, device='cuda'), torch.zeros(N, Fl, 2, device='cuda')
L.lstm_gates_fwd(pre, N, P, Fl, c0, g1, b1, g2, b2, c1, [(h.data_ptr(), Fl)], s1, s2)
dpre, dc0 = torch.zeros_like(pre), torch.zeros_like(c0)
dgs = [torch.zeros(4 * Fl, device='cuda'), torch.zeros(4 * Fl, device='cuda'), torch.zeros(Fl, device='cuda'), torch.zeros(Fl, device='cuda')]
L.lstm_gates_bwd(pre, N, P, Fl, c0, g1, b1, g2, b2, s1, s2, [(h.data_ptr(), Fl)], None, dpre, dc0, dgs[0], dgs[1], dgs[2], dgs[3])
torch.cuda.synchronize()
print('slab gates fwd/bwd: finite %s' % bool(torch.isfinite(dpre).all() and torch.isfinite(h).all()))
ok &= bool(torch.isfinite(dpre).all() and torch.isfinite(h).all())
# full-batch plane shapes: the planner picks clusters of 4 with 256 / 1024 positions per CTA (gates backward re-reading its
# pre-activations, 512-thread gates forward, two-pass instance-norm backward)
N = 32
pre, c0 = rnd(N, P, 4 * Fl), rnd(N, P, Fl, seed=3)
c1, h = torch.zeros(N, P, Fl, device='cuda'), torch.zeros(N, P, Fl, device='cuda')
s1, s2 = torch.zeros(N, 4 * Fl, 2, device='cuda'), torch.zeros(N, Fl, 2, device='cuda')
L.lstm_gates_fwd(pre, N, P, Fl, c0, g1, b1, g2, b2, c1, [(h.data_ptr(), Fl)], s1, s2)
dpre, dc0 = torch.zeros_like(pre), torch.zeros_like(c0)
L.lstm_gates_bwd(pre, N, P, Fl, c0, g1, b1, g2, b2, s1, s2, [(h.data_ptr(), Fl)], None, dpre, dc0, dgs[0], dgs[1], dgs[2], dgs[3])
x4, dy4 = rnd(N, 4096, C) + 1.0, rnd(N, 4096, C, seed=5)
y4, st4, dx4 = torch.zeros_like(x4), torch.zeros(N, C, 2, device='cuda'), torch.zeros_like(x4)
L.inorm_act(x4.data_ptr(), C, y4.data_ptr(), C, N, 4096, C, g, b, L.ACT_RELU, 0.0, st4)
dg4, db4 = torch.zeros(C, device='cuda'), torch.zeros(C, device='cuda')
L.inorm_act_bwd(x4.data_ptr(), C, [(dy4.data_ptr(), C)], dx4.data_ptr(), C, N, 4096, C, g, b, st4, L.ACT_RELU, 0.0, dg4, db4)
torch.cuda.synchronize()
fin = bool(torch.isfinite(dpre).all() and torch.isfinite(h).all() and torch.isfinite(dx4).all())
print('full-batch slab kernels (gates fwd/bwd 32x1024x32, instance norm fwd/bwd 32x4096x32): finite %s' % fin)
ok &= fin
# first discriminator layer on the tensor cores (csrc/d0_layer.cu) against the CUDA-core kernels
n, d, hh, ww, ci = 2, 3, 8, 64, 3
xv = torch.zeros(n, d, hh, ww, 4, device='cuda')
xv[..., :ci] = torch.rand(n, d, hh, ww, ci, device='cuda')
wv, bv, sig = rnd(3, 3, 3, ci, 32, seed=7, scale=0.2), rnd(32, seed=8), torch.tensor([1.3], device='cuda')
o1, o2 = torch.zeros(n, d, hh, ww, 32, device='cuda'), torch.zeros(n, d, hh, ww, 32, device='cuda')
L.conv3d_c4_fwd_tc(xv, wv, sig, bv, o1, n, d, hh, ww, ci, 0.1)
L.conv3d_c4_fwd(xv, wv, sig, bv, o2, n, d, hh, ww, ci, 0.1)
gw1, gw2 = torch.zeros(27 * ci * 32, device='cuda'), torch.zeros(27 * ci * 32, device='cuda')
L.check(L.lib().vp_conv3d_c4_wgrad_tc(L.ptr(xv), L.ptr(o2), L.ptr(gw1), n, d, hh, ww, ci, L.stream_ptr()))
gw3 = torch.zeros_like(gw1)
L.check(L.lib().vp_conv3d_c4_wgrad_tc(L.ptr(xv), L.ptr(o2), L.ptr(gw3), n, d, hh, ww, ci, L.stream_ptr()))
L.check(L.lib().vp_conv3d_c4_wgrad(L.ptr(xv), L.ptr(o2), L.ptr(gw2), n, d, hh, ww, ci, L.stream_ptr()))
torch.cuda.synchronize()
e1 = (o1 - o2).abs().max().item() / o2.abs().max().item()
e2 = ((gw1 - gw2).norm() / gw2.norm()).item()
print('first layer on tensor cores vs CUDA cores: forward rel %.1e, weight gradient rel L2 %.1e' % (e1, e2))
same = bool(torch.equal(gw1, gw3))
print('first-layer tensor-core weight gradient: two runs bit-identical %s' % same)
ok &= e1 < 3e-3 and e2 < 3e-3 and same
# table-driven weight packing, register-tiled wide dense layer, float4 cosine distance
wq = rnd(1, 5, 5, 72, 128, seed=9, scale=0.05)[0]
ref, n_pad, kc = L.pack_weights(wq, (1, 5, 5), 72, 128, L.WKIND_PLAIN, L.WLAYOUT_FWD)
outp = torch.zeros_like(ref)
L.PackPlan([(wq, (1, 5, 5), 72, 128, L.WKIND_PLAIN, L.WLAYOUT_FWD, None, None, None, outp)]).run()
xd_, wd_, bd_ = rnd(32, 2048), rnd(2048, 100, seed=1, scale=0.05), rnd(100, seed=2)
yd = torch.zeros(32, 100, device='cuda')
L.dense_fwd(xd_, 2048, wd_, bd_, yd, 100, 32, 2048, 100, k_splits=32)
dxd, dwd, dbd = torch.zeros_like(xd_), torch.zeros_like(wd_), torch.zeros_like(bd_)
L.dense_bwd(xd_, 2048, wd_, yd, 100, 32, 2048, 100, dx=dxd, dx_stride=2048, dw=dwd, dbias=dbd)
ca, cb = rnd(1000, 32), rnd(1000, 32, seed=1)
cda, cout_ = torch.zeros_like(ca), torch.zeros(1, device='cuda')
L.cosine_distance(ca, cb, cda, 1000, 32, 1.0, cout_)
torch.cuda.synchronize()
e3 = (yd.double() - (xd_.double() @ wd_.double() + bd_.double())).abs().max().item()
print('batched pack equal %s, wide dense max err %.1e, cosine distance finite %s' % (bool(torch.equal(outp, ref)), e3, bool(torch.isfinite(cda).all())))
ok &= bool(torch.equal(outp, ref)) and e3 < 1e-3 and bool(torch.isfinite(cda).all())
print('SANITIZE TARGET %s' % ('OK' if ok else 'MISMATCH'))
