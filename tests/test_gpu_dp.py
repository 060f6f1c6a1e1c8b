"""Data parallelism through the model's own API on real GPUs (needs >= 2: `gpurun --gpus 2 -- python -m pytest tests/test_gpu_dp.py -m gpu`):
the reference's multi-GPU semantics (base_model.py:517-646, tf_utils.py:450-480) -- the global batch split over `num_gpus`
towers, gradients averaged, every replica applying the same update -- must give what ONE GPU computes on the whole batch."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

HK = dict(context_frames=2, sequence_length=6, clip_length=4, lr=2e-4, beta1=0.5, l1_weight=100., kl_weight=1.0,
          video_sn_vae_gan_weight=0.1, video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0, kl_anneal_steps=(0, 10))
BG, STEP = 4, 5


def _case():
    sys.path.insert(0, ROOT)
    from oracle import savp_oracle as O
    hp = O.make_hparams(**HK)
    params, _ = O.init_params(hp, (64, 64, 3), seed=0)
    inputs, noise = O.make_synthetic_inputs(hp, BG, (64, 64, 3))
    g = torch.Generator().manual_seed(3)
    sampling = torch.rand(hp.sequence_length - 1 - hp.context_frames, BG, generator=g) < 0.5
    binp = {'images': inputs['images'].permute(1, 0, 2, 3, 4).contiguous()}
    return params, binp, noise, sampling


def _run(num_gpus):
    from video_prediction_b200.models import get_model_class
    params, binp, noise, sampling = _case()
    model = get_model_class('savp')(mode='train', hparams_dict=HK, num_gpus=num_gpus)
    model.set_params(params)
    model.build_graph(binp)          # num_gpus > 1: the GLOBAL batch; the model takes its shard
    model.global_step = STEP
    model.train_step(binp, noise, sampling=sampling)
    torch.cuda.synchronize()
    lv = model.losses()
    return model, lv


def _worker(rank, world, port, q, env):
    os.environ.update(env)
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port),
                      CUDA_VISIBLE_DEVICES=','.join(str(i) for i in range(world)))
    sys.path.insert(0, ROOT)
    torch.cuda.set_device(rank)
    model, lv = _run(world)
    assert model.B == BG // world and model.world_size == world
    q.put((rank, model.g_flat.cpu(), model.d_flat.cpu(), (model.g_grad / world).cpu(), (model.d_grad / world).cpu(), lv))
    import torch.distributed as dist
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('mode,buckets,tol', [('exact', '0', 3e-3), ('tf32', '1', 2e-2)])
def test_two_ranks_equal_one_rank_on_the_global_batch(mode, buckets, tol):
    """exact: fp32-exact convolutions (VP_EXACT=1) -> the two runs differ by fp32 summation order only.  tf32: product arithmetic, where different tile / split-K decisions at B/2 flip
    operand truncations downstream (two correct TF32 runs differ by ~0.5 %); this variant also exercises the bucketed,
    overlapped all-reduce (VP_DP_BUCKETS=1)."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp
    env = dict(VP_EXACT='1' if mode == 'exact' else '0', VP_DP_BUCKETS=buckets)
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29600 + (os.getpid() + (7 if mode == 'exact' else 0)) % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, env)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=600) for _ in range(2)), key=lambda r: r[0])
    for p in procs:
        p.join(120)
    (_, g0, d0, gg0, dg0, l0), (_, g1, d1, gg1, dg1, l1) = res
    # replicas stay bit-identical: same averaged gradients, same Adam update (tf_utils.py:450-480, base_model.py:590-616)
    assert torch.equal(g0, g1) and torch.equal(d0, d1) and torch.equal(gg0, gg1) and torch.equal(dg0, dg1)
    assert l0 == l1                                            # losses() averages over the replicas (tf_utils.py:489-490)
    os.environ.pop('WORLD_SIZE', None)
    os.environ.pop('RANK', None)
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        ref, lref = _run(1)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    for name, got, want in (('generator', gg0, ref.g_grad.cpu()), ('discriminator', dg0, ref.d_grad.cpu())):
        rel = ((got.double() - want.double()).norm() / want.double().norm()).item()
        print('[%s] %s gradient: 2 ranks x B/2 vs 1 rank x B, relative L2 %.2e' % (mode, name, rel))
        assert rel <= tol, (name, rel)
    for k, v in lref.items():
        assert abs(l0[k] - v) <= 5e-3 * abs(v) + 1e-6, (k, l0[k], v)
