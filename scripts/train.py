#!/usr/bin/env python
"""Training driver with the reference's command line (scripts/train.py:30-61 of alexlee-gk/video_prediction) on the H100
SAVP path.  Same flags, same options.json / dataset_hparams.json / model_hparams.json side files, same progress print-out
(global step, image/sec, d_loss / g_loss and their terms, learning rate), same checkpoint cadence -- no TensorFlow:
`sess.run(train_op)` becomes `model.train_step(batch)`.

    python scripts/train.py --input_dir data/bair --dataset bair --model savp \
        --model_hparams_dict hparams/bair_action_free/ours_savp/model_hparams.json --output_dir logs/savp
    python scripts/train.py --input_dir none --dataset synthetic --model savp ...        (no input files)
    torchrun --nproc-per-node 8 scripts/train.py ... --model_hparams batch_size=128      (data parallel, global batch split)

Datasets: `bair` / `softmotion` and `kth` read the reference's TFRecords on the host (video_prediction_b200/datasets), `synthetic`
generates videos.  Outside the hot path (SURVEY.md 8f-4): TensorBoard summaries (the *_summary_freq flags are accepted and
inert), the long-sequence validation model."""
from __future__ import absolute_import, division, print_function

import argparse
import errno
import json
import os
import random
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def build_parser():
    parser = argparse.ArgumentParser()
    parser.add_argument("--input_dir", type=str, required=True, help="either a directory containing subdirectories "
                                                                     "train, val, test, etc, or a directory containing "
                                                                     "the tfrecords (ignored by --dataset synthetic)")
    parser.add_argument("--val_input_dir", type=str, help="directories containing the tfrecords. default: input_dir")
    parser.add_argument("--logs_dir", default='logs', help="ignored if output_dir is specified")
    parser.add_argument("--output_dir", help="output directory where json files, summary, model, gifs, etc are saved. "
                                             "default is logs_dir/model_fname, where model_fname consists of "
                                             "information from model and model_hparams")
    parser.add_argument("--output_dir_postfix", default="")
    parser.add_argument("--checkpoint", help="directory with checkpoint or checkpoint name (e.g. checkpoint_dir/model-200000)")
    parser.add_argument("--resume", action='store_true', help='resume from lastest checkpoint in output_dir.')

    parser.add_argument("--dataset", type=str, help="dataset class name")
    parser.add_argument("--dataset_hparams", type=str, help="a string of comma separated list of dataset hyperparameters")
    parser.add_argument("--dataset_hparams_dict", type=str, help="a json file of dataset hyperparameters")
    parser.add_argument("--model", type=str, help="model class name")
    parser.add_argument("--model_hparams", type=str, help="a string of comma separated list of model hyperparameters")
    parser.add_argument("--model_hparams_dict", type=str, help="a json file of model hyperparameters")

    parser.add_argument("--summary_freq", type=int, default=1000, help="accepted for compatibility (summaries are not built)")
    parser.add_argument("--image_summary_freq", type=int, default=5000, help="accepted for compatibility")
    parser.add_argument("--eval_summary_freq", type=int, default=25000, help="accepted for compatibility")
    parser.add_argument("--accum_eval_summary_freq", type=int, default=100000, help="accepted for compatibility")
    parser.add_argument("--progress_freq", type=int, default=100, help="display progress every progress_freq steps")
    parser.add_argument("--save_freq", type=int, default=5000, help="save frequence of model, 0 to disable")

    parser.add_argument("--aggregate_nccl", type=int, default=0, help="gradients are always aggregated with NCCL here")
    parser.add_argument("--gpu_mem_frac", type=float, default=0, help="accepted for compatibility")
    parser.add_argument("--seed", type=int)
    return parser


def default_output_dir(args):
    """train.py:69-84: logs_dir/model=<name>.<hparams with = and , replaced>"""
    list_depth, model_fname = 0, ''
    for t in ('model=%s,%s' % (args.model, args.model_hparams)):
        if t == '[':
            list_depth += 1
        if t == ']':
            list_depth -= 1
        if list_depth and t == ',':
            t = '..'
        if t in '=,':
            t = '.'
        if t in '[]':
            t = ''
        model_fname += t
    return os.path.join(args.logs_dir, model_fname) + args.output_dir_postfix


def resolve_options(args):
    """Everything train.py does before it touches a dataset or a model (train.py:63-122); returns the two hparams dicts."""
    if args.output_dir is None:
        args.output_dir = default_output_dir(args)
    if args.resume:
        if args.checkpoint:
            raise ValueError('resume and checkpoint cannot both be specified')
        args.checkpoint = args.output_dir
    dataset_hparams_dict, model_hparams_dict = {}, {}
    if args.dataset_hparams_dict:
        with open(args.dataset_hparams_dict) as f:
            dataset_hparams_dict.update(json.loads(f.read()))
    if args.model_hparams_dict:
        with open(args.model_hparams_dict) as f:
            model_hparams_dict.update(json.loads(f.read()))
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
    return dataset_hparams_dict, model_hparams_dict


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.seed is not None:
        np.random.seed(args.seed)
        random.seed(args.seed)
    dataset_hparams_dict, model_hparams_dict = resolve_options(args)

    rank = int(os.environ.get('RANK', '0'))
    world = int(os.environ.get('WORLD_SIZE', '1'))
    chief = rank == 0
    if chief:
        print('----------------------------------- Options ------------------------------------')
        for k, v in args._get_kwargs():
            print(k, "=", v)
        print('------------------------------------- End --------------------------------------')

    from video_prediction_b200 import datasets, models
    VideoDataset = datasets.get_dataset_class(args.dataset)
    train_dataset = VideoDataset(args.input_dir, mode='train', seed=args.seed, hparams_dict=dataset_hparams_dict,
                                 hparams=args.dataset_hparams)
    VideoPredictionModel = models.get_model_class(args.model)
    hparams_dict = dict(model_hparams_dict)
    hparams_dict.update({
        'context_frames': train_dataset.hparams.context_frames,
        'sequence_length': train_dataset.hparams.sequence_length,
        'repeat': train_dataset.hparams.time_shift,
    })
    import torch
    if world > 1:
        torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', '0')))
    model = VideoPredictionModel(hparams_dict=hparams_dict, hparams=args.model_hparams, aggregate_nccl=args.aggregate_nccl,
                                 num_gpus=world if world > 1 else None)
    if args.seed is not None:
        model.random_seed = args.seed
    batch_size = model.hparams.batch_size            # GLOBAL batch; split over the ranks like the reference's towers
    model.build_graph(train_dataset.make_batch(batch_size))
    model.use_cuda_graph = True

    if chief:
        if not os.path.exists(args.output_dir):
            os.makedirs(args.output_dir)
        with open(os.path.join(args.output_dir, "options.json"), "w") as f:
            f.write(json.dumps(vars(args), sort_keys=True, indent=4))
        with open(os.path.join(args.output_dir, "dataset_hparams.json"), "w") as f:
            f.write(json.dumps(train_dataset.hparams.values(), sort_keys=True, indent=4))
        with open(os.path.join(args.output_dir, "model_hparams.json"), "w") as f:
            f.write(json.dumps(model.hparams.values(), sort_keys=True, indent=4))
        print("parameter_count =", int(sum(int(np.prod(v.shape)) for k, v in model.params.items() if not k.endswith('/u'))))

    model.restore(None, args.checkpoint)
    start_step = model.global_step
    max_steps = model.hparams.max_steps

    def should(step, freq):
        if freq is None:
            return (step + 1) == (max_steps - start_step)
        return freq and ((step + 1) % freq == 0 or (step + 1) in (0, max_steps - start_step))

    start_time = time.time()
    for step in range(0, max_steps - start_step):
        if step == 1:
            start_time = time.time()         # skip step 0 for timing purposes (warm start, graph capture)
        global_step = model.global_step      # read before it is incremented, as the reference's fetch
        model.train_step(train_dataset.make_batch(batch_size))
        if should(step, args.progress_freq):
            model.losses()                   # device -> host (mean over replicas), refreshes g_loss / d_loss / ...
            if chief:
                steps_per_epoch = train_dataset.num_examples_per_epoch() / batch_size
                print("progress  global step %d  epoch %0.1f" % (global_step + 1, global_step / steps_per_epoch))
                if step > 0:
                    torch.cuda.synchronize()
                    average_time = (time.time() - start_time) / step
                    remaining_time = (max_steps - (start_step + step + 1)) * average_time
                    print("          image/sec %0.1f  remaining %dm (%0.1fh) (%0.1fd)" %
                          (batch_size / average_time, remaining_time / 60, remaining_time / 60 / 60, remaining_time / 60 / 60 / 24))
                if model.d_losses:
                    print("d_loss", model.d_loss)
                for name, loss in model.d_losses.items():
                    print("  ", name, loss)
                if model.g_losses:
                    print("g_loss", model.g_loss)
                for name, loss in model.g_losses.items():
                    print("  ", name, loss)
                print("learning_rate", model.learning_rate_at(global_step))
        if should(step, args.save_freq) and chief:
            print("saving model to", args.output_dir)
            model.save(args.output_dir)
            print("done")
    return model


if __name__ == '__main__':
    main()
