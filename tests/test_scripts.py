"""The reference's command lines run through scripts/train.py / scripts/generate.py (CPU part: argument set, option
resolution, side files; GPU part: three optimisation steps, a checkpoint, and sampling from it)."""
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

REFERENCE_TRAIN_FLAGS = ['--input_dir', '--val_input_dir', '--logs_dir', '--output_dir', '--output_dir_postfix', '--checkpoint',
                         '--resume', '--dataset', '--dataset_hparams', '--dataset_hparams_dict', '--model', '--model_hparams',
                         '--model_hparams_dict', '--summary_freq', '--image_summary_freq', '--eval_summary_freq',
                         '--accum_eval_summary_freq', '--progress_freq', '--save_freq', '--aggregate_nccl', '--gpu_mem_frac', '--seed']
REFERENCE_GENERATE_FLAGS = ['--input_dir', '--results_dir', '--results_gif_dir', '--results_png_dir', '--output_gif_dir',
                            '--output_png_dir', '--checkpoint', '--mode', '--dataset', '--dataset_hparams', '--model',
                            '--model_hparams', '--batch_size', '--num_samples', '--num_epochs', '--num_stochastic_samples',
                            '--gif_length', '--fps', '--gpu_mem_frac', '--seed']


def test_train_and_generate_accept_the_reference_argument_set(tmp_path):
    import train
    import generate
    flags = {a.option_strings[0]: a for a in train.build_parser()._actions if a.option_strings}
    assert set(REFERENCE_TRAIN_FLAGS) <= set(flags)                          # the reference's scripts/train.py:30-61
    assert flags['--summary_freq'].default == 1000 and flags['--save_freq'].default == 5000 and flags['--progress_freq'].default == 100
    gflags = {a.option_strings[0]: a for a in generate.build_parser()._actions if a.option_strings}
    assert set(REFERENCE_GENERATE_FLAGS) <= set(gflags)                      # the reference's scripts/generate.py:19-49
    assert gflags['--batch_size'].default == 8 and gflags['--num_stochastic_samples'].default == 5 and gflags['--seed'].default == 7
    # the README's training command line (bair_action_free / ours_savp), with the synthetic dataset
    hp = tmp_path / 'model_hparams.json'
    hp.write_text(json.dumps(dict(batch_size=16, lr=0.0002, beta1=0.5, l1_weight=100.0, kl_weight=1.0, video_sn_vae_gan_weight=0.1,
                                  video_sn_gan_weight=0.1, vae_gan_feature_cdist_weight=10.0)))
    args = train.build_parser().parse_args(['--input_dir', 'data/bair', '--dataset', 'synthetic', '--model', 'savp',
                                            '--model_hparams_dict', str(hp), '--model_hparams', 'kernel_size=[5,5],lr=0.001',
                                            '--logs_dir', str(tmp_path)])
    d, m = train.resolve_options(args)
    assert m['l1_weight'] == 100.0 and d == {}
    assert args.output_dir == os.path.join(str(tmp_path), 'model.savp.kernel_size.5..5.lr.0.001')   # train.py:69-84
    with pytest.raises(ValueError):
        a = train.build_parser().parse_args(['--input_dir', 'x', '--resume', '--checkpoint', 'y'])
        train.resolve_options(a)
    with pytest.raises(ValueError):
        generate.resolve_options(generate.build_parser().parse_args(['--input_dir', 'x']))     # dataset required w/o checkpoint


def test_dataset_registry_and_synthetic_batches():
    from video_prediction_b200 import datasets
    with pytest.raises(ValueError, match='Invalid dataset'):
        datasets.get_dataset_class('bogus')
    with pytest.raises(NotImplementedError):
        datasets.get_dataset_class('google_robot')
    DS = datasets.get_dataset_class('synthetic')
    ds = DS('ignored', mode='val', num_epochs=1, seed=3, hparams='sequence_length=6,action_dim=4,num_examples=8')
    assert ds.hparams.long_sequence_length == 6 and ds.hparams.context_frames == 2
    b = ds.make_batch(4)
    assert b['images'].shape == (4, 6, 64, 64, 3) and b['images'].dtype == np.float32 and b['actions'].shape == (4, 5, 4)
    assert 0.0 <= b['images'].min() and b['images'].max() <= 1.0
    ds.make_batch(4)
    with pytest.raises(StopIteration):
        ds.make_batch(4)
    with pytest.raises(ValueError):
        DS('x', mode='bad')


@pytest.mark.gpu
def test_train_three_steps_checkpoint_resume_and_generate(tmp_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    import train
    import generate
    out = str(tmp_path / 'run')
    common = ['--input_dir', 'none', '--dataset', 'synthetic', '--dataset_hparams', 'sequence_length=6,num_examples=8',
              '--model', 'savp', '--output_dir', out, '--progress_freq', '1', '--save_freq', '3', '--seed', '1']
    hp = 'batch_size=2,max_steps=3,clip_length=4,lr=0.0002,beta1=0.5,l1_weight=100.0,kl_weight=1.0,video_sn_vae_gan_weight=0.1,' \
         'video_sn_gan_weight=0.1,vae_gan_feature_cdist_weight=10.0'
    model = train.main(common + ['--model_hparams', hp])
    assert model.global_step == 3 and model.g_loss is not None and np.isfinite(model.g_loss) and np.isfinite(model.d_loss)
    assert set(model.g_losses) >= {'gen_l1_loss', 'gen_video_sn_gan_loss'} and 'gen_kl_loss' not in model.g_losses  # KL weight 0 at step 2
    for f in ('options.json', 'dataset_hparams.json', 'model_hparams.json', 'checkpoint', 'model-3.npz'):
        assert os.path.exists(os.path.join(out, f)), f
    w = model.get_params()['generator/rnn/savp_cell/h0/conv_pool2d/kernel']
    # resume: options / hparams come from the checkpoint directory, training continues at step 3
    model2 = train.main(['--input_dir', 'none', '--output_dir', out, '--resume', '--model_hparams', 'max_steps=4',
                         '--progress_freq', '1', '--save_freq', '0'])
    assert model2.global_step == 4 and model2.g_adam_t == 4
    assert model2.hparams.l1_weight == 100.0 and model2.hparams.clip_length == 4
    # sampling from the checkpoint
    n = generate.main(['--input_dir', 'none', '--checkpoint', out, '--results_dir', str(tmp_path / 'results'), '--batch_size', '2',
                       '--num_samples', '2', '--num_stochastic_samples', '2', '--mode', 'test'])
    assert n == 2
    png_dir = str(tmp_path / 'results' / 'run')
    pngs = [p for p in os.listdir(png_dir) if p.endswith('.png')]
    assert len(pngs) == 2 * 2 * 4                                           # samples x stochastic samples x future frames
    from PIL import Image
    gif = Image.open(os.path.join(png_dir, 'gen_image_00000_00.gif'))
    assert gif.n_frames == 6 and gif.size == (64, 64)                       # context + future frames, --fps 4
    a = np.load(os.path.join(png_dir, 'gen_image_00000_00.npy'))
    b = np.load(os.path.join(png_dir, 'gen_image_00000_01.npy'))
    assert a.shape == (6, 64, 64, 3) and a.dtype == np.uint8
    assert np.array_equal(a[:2], b[:2]) and not np.array_equal(a[2:], b[2:])    # same context, different noise draws
    # a TensorFlow-format checkpoint (tensor bundle) of the same variables, with the historical 'dna_cell' scope and Adam slots:
    # restore() reads it through tf_checkpoint.py and the savp_cell -> dna_cell mapping (savp_model.py:848-855)
    from test_tf_checkpoint import write_bundle
    tensors = {k.replace('savp_cell', 'dna_cell'): v for k, v in model2.get_params().items()}
    k0 = 'generator/rnn/savp_cell/h0/conv_pool2d/kernel'
    tensors[k0.replace('savp_cell', 'dna_cell') + '/Adam'] = np.full(w.shape, 0.25, np.float32)
    tensors['global_step'] = np.array(1234, np.int64)
    tensors['beta1_power'] = np.array(0.5 ** 6, np.float32)
    tf_dir = tmp_path / 'tf_ckpt'
    tf_dir.mkdir()
    write_bundle(str(tf_dir / 'model-1234'), tensors)
    (tf_dir / 'checkpoint').write_text('model_checkpoint_path: "model-1234"\n')
    from video_prediction_b200.models import get_model_class
    m3 = get_model_class('savp')(mode='train', hparams_dict=model2.hparams.values())
    m3.build_graph({'images': np.zeros((2, 6, 64, 64, 3), np.float32)})
    m3.restore(None, str(tf_dir))
    assert m3.global_step == 1234 and m3.g_adam_t == 5
    for k, v in model2.get_params().items():
        assert np.array_equal(m3.get_params()[k], v), k
    assert float(m3._view_of(m3.g_m, m3.g_flat, k0).mean()) == 0.25
    # best-of-N evaluation (base_model.py:132-227): 3 stochastic samples, psnr / mse / ssim min / avg / max per video
    m4 = get_model_class('savp')(mode='test', hparams_dict=model2.hparams.values())
    from video_prediction_b200 import datasets
    batch = datasets.get_dataset_class('synthetic')('none', mode='test', seed=5, hparams='sequence_length=6').make_batch(2)
    m4.build_graph(batch)
    m4.restore(None, out)
    eo, em = m4.eval_outputs_and_metrics(batch, num_samples=3)
    assert tuple(em['eval_psnr/max'].shape) == (2, 4) and tuple(eo['eval_gen_images_ssim/max'].shape) == (2, 5, 64, 64, 3)
    for name in ('psnr', 'ssim'):
        lo, av, hi = (em['eval_%s/%s' % (name, k)].mean(dim=1) for k in ('min', 'avg', 'max'))
        assert bool((lo <= av + 1e-6).all()) and bool((av <= hi + 1e-6).all()) and bool((hi > lo).any())
    assert bool((em['eval_mse/min'] >= 0).all()) and float(em['eval_ssim/max'].max()) <= 1.0


@pytest.mark.gpu
def test_train_on_bair_format_tfrecords_with_actions(tmp_path):
    """scripts/train.py --dataset bair: TFRecords in the BAIR layout (one Example per trajectory, raw 64x64x3 frames,
    4-d actions, 3-d states) -> host pipeline (datasets/video_datasets.py) -> action-conditioned SAVP training steps."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    import train
    from video_prediction_b200.datasets import tfrecord as R
    rng = np.random.default_rng(0)
    d = tmp_path / 'bair' / 'train'
    d.mkdir(parents=True)
    recs = []
    for k in range(4):
        base = rng.integers(0, 255, (64, 64, 3), dtype=np.uint8)
        f = {}
        for t in range(30):
            f['%d/image_aux1/encoded' % t] = np.roll(base, (t, 2 * t), axis=(0, 1)).tobytes()
            f['%d/endeffector_pos' % t] = rng.standard_normal(3).astype(np.float32)
            if t < 29:
                f['%d/action' % t] = rng.standard_normal(4).astype(np.float32)
        recs.append(R.make_example(f))
    R.write_records(str(d / 'traj_0_to_3.tfrecords'), recs)
    out = str(tmp_path / 'run')
    model = train.main(['--input_dir', str(tmp_path / 'bair'), '--dataset', 'bair', '--dataset_hparams', 'use_state=True,sequence_length=6',
                        '--model', 'savp', '--output_dir', out, '--progress_freq', '1', '--save_freq', '0', '--seed', '2',
                        '--model_hparams', 'batch_size=2,max_steps=2,clip_length=4,l1_weight=100.0,kl_weight=1.0,video_sn_gan_weight=0.1'])
    assert model.global_step == 2 and np.isfinite(model.g_loss) and np.isfinite(model.d_loss)
    assert model.hparams.repeat == 2 and model.hparams.sequence_length == 6          # time_shift of the BAIR dataset (train.py:160)
    assert model.A == 4                                                              # actions reached the model


REFERENCE_EVALUATE_FLAGS = ['--input_dir', '--results_dir', '--output_dir', '--checkpoint', '--mode', '--dataset', '--dataset_hparams',
                            '--model', '--model_hparams', '--batch_size', '--num_samples', '--num_epochs', '--eval_substasks',
                            '--only_metrics', '--num_stochastic_samples', '--gt_inputs_dir', '--gt_outputs_dir',
                            '--eval_parallel_iterations', '--gpu_mem_frac', '--seed']


def test_evaluate_accepts_the_reference_argument_set_and_writes_its_csv_layout(tmp_path):
    import evaluate
    flags = {a.option_strings[0]: a for a in evaluate.build_parser()._actions if a.option_strings}
    assert set(REFERENCE_EVALUATE_FLAGS) <= set(flags)                       # the reference's scripts/evaluate.py:143-175
    assert flags['--num_stochastic_samples'].default == 100 and flags['--eval_substasks'].default == ['max', 'avg', 'min']
    assert flags['--mode'].choices == ['val', 'test'] and flags['--seed'].default == 7
    with pytest.raises(ValueError):
        evaluate.resolve_options(evaluate.build_parser().parse_args(['--input_dir', 'x', '--model', 'savp']))
    a = evaluate.build_parser().parse_args(['--input_dir', 'x', '--model', 'savp', '--dataset', 'synthetic', '--results_dir', str(tmp_path)])
    evaluate.resolve_options(a)
    assert a.output_dir == os.path.join(str(tmp_path), 'model.savp')
    # metrics files: header + appended batches, read back without index / mean columns (evaluate.py:44-66)
    m0, m1 = np.arange(6, dtype=np.float32).reshape(2, 3), np.arange(6, 12, dtype=np.float32).reshape(2, 3)
    fname = str(tmp_path / 'task' / 'metrics' / 'psnr')
    evaluate.save_metrics(fname, m0, 0)
    evaluate.save_metrics(fname, m1, 2)
    rows = open(fname + '.csv').read().splitlines()
    assert rows[0].split('\t') == ['sample_ind', '0', '1', '2', 'mean'] and rows[3].split('\t')[0] == '2' and len(rows) == 5
    assert np.array_equal(evaluate.load_metrics(fname), np.concatenate([m0, m1]))


@pytest.mark.gpu
def test_evaluate_best_of_n_on_a_trained_checkpoint(tmp_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    import train
    import evaluate
    out = str(tmp_path / 'run')
    train.main(['--input_dir', 'none', '--dataset', 'synthetic', '--dataset_hparams', 'sequence_length=6,num_examples=8', '--model', 'savp',
                '--output_dir', out, '--progress_freq', '0', '--save_freq', '2', '--seed', '1',
                '--model_hparams', 'batch_size=2,max_steps=2,clip_length=4,l1_weight=100.0,kl_weight=1.0,video_sn_gan_weight=0.1'])
    res = str(tmp_path / 'results')
    summary = evaluate.main(['--input_dir', 'none', '--checkpoint', out, '--mode', 'test', '--results_dir', res, '--batch_size', '2',
                             '--num_samples', '4', '--num_stochastic_samples', '3'])
    assert set(summary) == {'psnr', 'ssim', 'mse'} and all(np.isfinite(v) for v in summary.values())
    base = os.path.join(res, 'run')
    for metric in ('psnr', 'ssim', 'mse'):
        best = evaluate.load_metrics(os.path.join(base, 'prediction_eval_%s_max' % metric, 'metrics', metric))
        avg = evaluate.load_metrics(os.path.join(base, 'prediction_eval_%s_avg' % metric, 'metrics', metric))
        worst = evaluate.load_metrics(os.path.join(base, 'prediction_eval_%s_min' % metric, 'metrics', metric))
        assert best.shape == (4, 4)                                          # 4 videos x 4 future frames
        assert (best.mean(1) >= avg.mean(1) - 1e-6).all() and (avg.mean(1) >= worst.mean(1) - 1e-6).all()
    pngs = os.listdir(os.path.join(base, 'prediction_eval_psnr_max', 'outputs'))
    assert len(pngs) == 4 * 4 and len(os.listdir(os.path.join(base, 'prediction_eval_psnr_max', 'inputs'))) == 4 * 2
