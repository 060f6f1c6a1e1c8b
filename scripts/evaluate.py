#!/usr/bin/env python
"""Evaluation driver with the reference's command line (scripts/evaluate.py:143-175 of alexlee-gk/video_prediction) on the H100
SAVP path: for every batch of the val / test split, `num_stochastic_samples` predictions are drawn and the best / average /
worst one per video is kept for every metric (base_model.py:132-227 -> `model.eval_outputs_and_metrics`), written in the
reference's result layout

    <output_dir>/prediction_eval_<metric>_<subtask>/metrics/<metric>.csv        tab-separated: sample_ind, one column per future frame, mean
    <output_dir>/prediction_eval_<metric>_<subtask>/inputs/context_image_<sample>_<t>.png
    <output_dir>/prediction_eval_<metric>_<subtask>/outputs/gen_image_<sample>_<t>.png

and summarised per time step (mean (std)) at the end.  Metrics: psnr, ssim, mse (video_prediction_b200/metrics.py, tf.image
semantics); lpips needs downloaded network weights and is absent (SURVEY.md 8f-2).

    python scripts/evaluate.py --input_dir data/bair --dataset_hparams sequence_length=30 --checkpoint logs/savp \\
        --mode test --results_dir results --batch_size 8 --num_stochastic_samples 100"""
from __future__ import absolute_import, division, print_function

import argparse
import csv
import errno
import json
import os
import random
import re
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def build_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--input_dir", type=str, required=True, help="either a directory containing subdirectories train, val, test, "
                                                                "etc, or a directory containing the tfrecords")
    p.add_argument("--results_dir", type=str, default='results', help="ignored if output_dir is specified")
    p.add_argument("--output_dir", help="output directory where results are saved. default is results_dir/model_fname, "
                                        "where model_fname is the directory name of checkpoint")
    p.add_argument("--checkpoint", help="directory with checkpoint or checkpoint name (e.g. checkpoint_dir/model-200000)")
    p.add_argument("--mode", type=str, choices=['val', 'test'], default='val', help='mode for dataset, val or test.')
    p.add_argument("--dataset", type=str, help="dataset class name")
    p.add_argument("--dataset_hparams", type=str, help="a string of comma separated list of dataset hyperparameters")
    p.add_argument("--model", type=str, help="model class name")
    p.add_argument("--model_hparams", type=str, help="a string of comma separated list of model hyperparameters")
    p.add_argument("--batch_size", type=int, default=8, help="number of samples in batch")
    p.add_argument("--num_samples", type=int, help="number of samples in total (all of them by default)")
    p.add_argument("--num_epochs", type=int, default=1)
    p.add_argument("--eval_substasks", type=str, nargs='+', default=['max', 'avg', 'min'], help='subtasks to evaluate (e.g. max, avg, min)')
    p.add_argument("--only_metrics", action='store_true')
    p.add_argument("--num_stochastic_samples", type=int, default=100)
    p.add_argument("--gt_inputs_dir", type=str, help="accepted for compatibility (ismple dataset), unused")
    p.add_argument("--gt_outputs_dir", type=str, help="accepted for compatibility (ismple dataset), unused")
    p.add_argument("--eval_parallel_iterations", type=int, default=10, help="accepted for compatibility (tf.map_fn), unused")
    p.add_argument("--gpu_mem_frac", type=float, default=0, help="accepted for compatibility, unused")
    p.add_argument("--seed", type=int, default=7)
    return p


def resolve_options(args):
    """Options and hparams stored next to the checkpoint (evaluate.py:183-210)."""
    dataset_hparams_dict, model_hparams_dict = {}, {}
    if args.checkpoint:
        checkpoint_dir = os.path.normpath(args.checkpoint)
        if not os.path.isdir(args.checkpoint):
            checkpoint_dir, _ = os.path.split(checkpoint_dir)
        if not os.path.exists(checkpoint_dir):
            raise FileNotFoundError(errno.ENOENT, os.strerror(errno.ENOENT), checkpoint_dir)
        with open(os.path.join(checkpoint_dir, "options.json")) as f:
            print("loading options from checkpoint %s" % args.checkpoint)
            options = json.loads(f.read())
            args.dataset = args.dataset or options['dataset']
            args.model = args.model or options['model']
        for fname, target in (("dataset_hparams.json", dataset_hparams_dict), ("model_hparams.json", model_hparams_dict)):
            try:
                with open(os.path.join(checkpoint_dir, fname)) as f:
                    target.update(json.loads(f.read()))
            except FileNotFoundError:
                print("%s was not loaded because it does not exist" % fname)
        args.output_dir = args.output_dir or os.path.join(args.results_dir, os.path.split(checkpoint_dir)[1])
    else:
        if not args.dataset:
            raise ValueError('dataset is required when checkpoint is not specified')
        if not args.model:
            raise ValueError('model is required when checkpoint is not specified')
        args.output_dir = args.output_dir or os.path.join(args.results_dir, 'model.%s' % args.model)
    return dataset_hparams_dict, model_hparams_dict


def save_metrics(prefix_fname, metrics, sample_start_ind=0):
    os.makedirs(os.path.dirname(prefix_fname), exist_ok=True)
    assert metrics.ndim == 2
    with open('%s.csv' % prefix_fname, 'w' if sample_start_ind == 0 else 'a', newline='') as f:
        w = csv.writer(f, delimiter='\t', quotechar='|', quoting=csv.QUOTE_MINIMAL)
        if sample_start_ind == 0:
            w.writerow(['sample_ind'] + [str(t) for t in range(metrics.shape[1])] + ['mean'])
        for i, row in enumerate(metrics):
            w.writerow([str(sample_start_ind + i)] + [str(v) for v in row] + [str(np.mean(row))])


def load_metrics(prefix_fname):
    with open('%s.csv' % prefix_fname, newline='') as f:
        rows = list(csv.reader(f, delimiter='\t', quotechar='|'))
    return np.array(rows)[1:, 1:-1].astype(np.float32)          # without the header, the index column and the mean column


def save_image_sequences(prefix_fname, videos, sample_start_ind=0):
    import cv2
    os.makedirs(os.path.dirname(prefix_fname), exist_ok=True)
    for i, video in enumerate(videos):
        for t, image in enumerate(video):
            image = (np.clip(image, 0.0, 1.0) * 255.0).astype(np.uint8)
            image = np.tile(image, (1, 1, 3)) if image.shape[-1] == 1 else cv2.cvtColor(image, cv2.COLOR_RGB2BGR)
            cv2.imwrite('%s_%05d_%02d.png' % (prefix_fname, sample_start_ind + i, t), image)


def save_prediction_eval_results(task_dir, results, hparams, sample_start_ind, only_metrics, subtasks):
    future = hparams.sequence_length - hparams.context_frames
    context_images = results['eval_images'][:, :hparams.context_frames]
    for subtask in subtasks:
        for key in list(results):
            m = re.match(r'eval_(\w+)/%s$' % subtask, key)
            if not m or key.startswith('eval_gen_images_'):
                continue
            name = m.group(1)
            subtask_dir = task_dir + '_%s_%s' % (name, subtask)
            save_metrics(os.path.join(subtask_dir, 'metrics', name), results[key], sample_start_ind)
            if only_metrics:
                continue
            gen = results.get('eval_gen_images_%s/%s' % (name, subtask), results.get('eval_gen_images'))
            save_image_sequences(os.path.join(subtask_dir, 'inputs', 'context_image'), context_images, sample_start_ind)
            save_image_sequences(os.path.join(subtask_dir, 'outputs', 'gen_image'), gen[:, -future:], sample_start_ind)


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.seed is not None:
        np.random.seed(args.seed)
        random.seed(args.seed)
    dataset_hparams_dict, model_hparams_dict = resolve_options(args)
    print('----------------------------------- Options ------------------------------------')
    for k, v in args._get_kwargs():
        print(k, "=", v)
    print('------------------------------------- End --------------------------------------')

    from video_prediction_b200 import datasets, models
    dataset = datasets.get_dataset_class(args.dataset)(args.input_dir, mode=args.mode, num_epochs=args.num_epochs, seed=args.seed,
                                                       hparams_dict=dataset_hparams_dict, hparams=args.dataset_hparams)
    hparams_dict = dict(model_hparams_dict)
    hparams_dict.update({'context_frames': dataset.hparams.context_frames, 'sequence_length': dataset.hparams.sequence_length,
                         'repeat': dataset.hparams.time_shift})
    model = models.get_model_class(args.model)(mode=args.mode, hparams_dict=hparams_dict, hparams=args.model_hparams,
                                               eval_num_samples=args.num_stochastic_samples,
                                               eval_parallel_iterations=args.eval_parallel_iterations)
    if args.num_samples:
        if args.num_samples > dataset.num_examples_per_epoch():
            raise ValueError('num_samples cannot be larger than the dataset')
        num_examples_per_epoch = args.num_samples
    else:
        num_examples_per_epoch = dataset.num_examples_per_epoch()
    if num_examples_per_epoch % args.batch_size != 0:
        raise ValueError('batch_size should evenly divide the dataset size %d' % num_examples_per_epoch)

    inputs = dataset.make_batch(args.batch_size)
    model.build_graph(inputs)
    os.makedirs(args.output_dir, exist_ok=True)
    for fname, content in (("options.json", vars(args)), ("dataset_hparams.json", dataset.hparams.values()),
                           ("model_hparams.json", model.hparams.values())):
        with open(os.path.join(args.output_dir, fname), "w") as f:
            f.write(json.dumps(content, sort_keys=True, indent=4))
    model.restore(None, args.checkpoint)

    sample_ind = 0
    while not (args.num_samples and sample_ind >= args.num_samples):
        if sample_ind > 0:
            try:
                inputs = dataset.make_batch(args.batch_size)
            except StopIteration:                                 # tf.errors.OutOfRangeError in the reference
                break
        print("evaluation samples from %d to %d" % (sample_ind, sample_ind + args.batch_size))
        eval_outputs, eval_metrics = model.eval_outputs_and_metrics(inputs, noise_seed=args.seed or 0)
        results = {k: v.detach().cpu().numpy() for k, v in list(eval_outputs.items()) + list(eval_metrics.items())}
        save_prediction_eval_results(os.path.join(args.output_dir, 'prediction_eval'), results, model.hparams, sample_ind,
                                     args.only_metrics, args.eval_substasks)
        sample_ind += args.batch_size

    summary = {}
    for metric_name in ('psnr', 'ssim', 'mse'):
        fname = os.path.join(args.output_dir, 'prediction_eval_%s_max' % metric_name, 'metrics', metric_name)
        if not os.path.exists(fname + '.csv'):
            continue
        metric = load_metrics(fname)
        summary[metric_name] = float(metric.mean())
        print('=' * 31)
        print('prediction_eval_%s_max' % metric_name, metric_name)
        print('-' * 31)
        print('{:>10} {:>20}'.format('time step', metric_name))
        for t, (mean, std) in enumerate(zip(metric.mean(axis=0), metric.std(axis=0))):
            print('{:>10} {:>10.4f} ({:>7.4f})'.format(t, mean, std))
        print('{:>10} {:>10.4f} ({:>7.4f})'.format('mean (std)', metric.mean(), metric.std()))
        print('=' * 31)
    return summary


if __name__ == '__main__':
    main()
