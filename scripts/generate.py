#!/usr/bin/env python
"""Sampling driver with the reference's command line (scripts/generate.py:19-49) on the H100 SAVP path: restores a
checkpoint written by scripts/train.py, runs the generator in test mode (prior unroll, no discriminators) for
`--num_stochastic_samples` noise draws per batch, and writes the predicted future frames as PNGs
(`gen_image_%05d_%02d_%02d.png`, generate.py:183-190) and, per sample, the context + future frames as an animated GIF
`<output_gif_dir>/gen_image_%05d_%02d.gif` at `--fps` (generate.py:176-181; written with PIL instead of the reference's
moviepy / ffmpeg) next to the same frames as `gen_image_%05d_%02d.npy`, [context + future, H, W, C] uint8."""
from __future__ import absolute_import, division, print_function

import argparse
import errno
import json
import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def build_parser():
    parser = argparse.ArgumentParser()
    parser.add_argument("--input_dir", type=str, required=True, help="either a directory containing subdirectories "
                                                                     "train, val, test, etc, or a directory containing "
                                                                     "the tfrecords (ignored by --dataset synthetic)")
    parser.add_argument("--results_dir", type=str, default='results', help="ignored if output_gif_dir is specified")
    parser.add_argument("--results_gif_dir", type=str, help="default is results_dir. ignored if output_gif_dir is specified")
    parser.add_argument("--results_png_dir", type=str, help="default is results_dir. ignored if output_png_dir is specified")
    parser.add_argument("--output_gif_dir", help="output directory where samples are saved as frame stacks. default is "
                                                 "results_gif_dir/model_fname")
    parser.add_argument("--output_png_dir", help="output directory where samples are saved as pngs. default is "
                                                 "results_png_dir/model_fname")
    parser.add_argument("--checkpoint", help="directory with checkpoint or checkpoint name (e.g. checkpoint_dir/model-200000)")
    parser.add_argument("--mode", type=str, choices=['val', 'test'], default='val', help='mode for dataset, val or test.')
    parser.add_argument("--dataset", type=str, help="dataset class name")
    parser.add_argument("--dataset_hparams", type=str, help="a string of comma separated list of dataset hyperparameters")
    parser.add_argument("--model", type=str, help="model class name")
    parser.add_argument("--model_hparams", type=str, help="a string of comma separated list of model hyperparameters")
    parser.add_argument("--batch_size", type=int, default=8, help="number of samples in batch")
    parser.add_argument("--num_samples", type=int, help="number of samples in total (all of them by default)")
    parser.add_argument("--num_epochs", type=int, default=1)
    parser.add_argument("--num_stochastic_samples", type=int, default=5)
    parser.add_argument("--gif_length", type=int, help="default is sequence_length")
    parser.add_argument("--fps", type=int, default=4)
    parser.add_argument("--gpu_mem_frac", type=float, default=0, help="accepted for compatibility")
    parser.add_argument("--seed", type=int, default=7)
    return parser


def resolve_options(args):
    """generate.py:57-90."""
    args.results_gif_dir = args.results_gif_dir or args.results_dir
    args.results_png_dir = args.results_png_dir or args.results_dir
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
        try:
            with open(os.path.join(checkpoint_dir, "dataset_hparams.json")) as f:
                dataset_hparams_dict = json.loads(f.read())
        except FileNotFoundError:
            print("dataset_hparams.json was not loaded because it does not exist")
        try:
            with open(os.path.join(checkpoint_dir, "model_hparams.json")) as f:
                model_hparams_dict = json.loads(f.read())
        except FileNotFoundError:
            print("model_hparams.json was not loaded because it does not exist")
        args.output_gif_dir = args.output_gif_dir or os.path.join(args.results_gif_dir, os.path.split(checkpoint_dir)[1])
        args.output_png_dir = args.output_png_dir or os.path.join(args.results_png_dir, os.path.split(checkpoint_dir)[1])
    else:
        if not args.dataset:
            raise ValueError('dataset is required when checkpoint is not specified')
        if not args.model:
            raise ValueError('model is required when checkpoint is not specified')
        args.output_gif_dir = args.output_gif_dir or os.path.join(args.results_gif_dir, 'model.%s' % args.model)
        args.output_png_dir = args.output_png_dir or os.path.join(args.results_png_dir, 'model.%s' % args.model)
    return dataset_hparams_dict, model_hparams_dict


def save_gif(path, frames, fps):
    """Animated GIF of uint8 frames [H,W,C] (C = 1 or 3); utils/ffmpeg_gif.py:save_gif in the reference."""
    try:
        from PIL import Image
    except ImportError:                               # the frame stack (.npy) is still written
        return False
    imgs = [Image.fromarray(f[..., 0] if f.shape[-1] == 1 else f) for f in frames]
    imgs[0].save(path, save_all=True, append_images=imgs[1:], duration=int(round(1000.0 / max(fps, 1))), loop=0)
    return True


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
    VideoDataset = datasets.get_dataset_class(args.dataset)
    dataset = VideoDataset(args.input_dir, mode=args.mode, num_epochs=args.num_epochs, seed=args.seed,
                           hparams_dict=dataset_hparams_dict, hparams=args.dataset_hparams)
    VideoPredictionModel = models.get_model_class(args.model)
    hparams_dict = dict(model_hparams_dict)
    hparams_dict.update({'context_frames': dataset.hparams.context_frames, 'sequence_length': dataset.hparams.sequence_length,
                         'repeat': 1 if args.dataset in ('synthetic', 'SyntheticVideoDataset') else dataset.hparams.time_shift})
    model = VideoPredictionModel(mode=args.mode, hparams_dict=hparams_dict, hparams=args.model_hparams)
    model.random_seed = args.seed or 0
    sequence_length, context_frames = model.hparams.sequence_length, model.hparams.context_frames
    future_length = sequence_length - context_frames

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
    for output_dir in (args.output_gif_dir, args.output_png_dir):
        if not os.path.exists(output_dir):
            os.makedirs(output_dir)
        with open(os.path.join(output_dir, "options.json"), "w") as f:
            f.write(json.dumps(vars(args), sort_keys=True, indent=4))
        with open(os.path.join(output_dir, "dataset_hparams.json"), "w") as f:
            f.write(json.dumps(dataset.hparams.values(), sort_keys=True, indent=4))
        with open(os.path.join(output_dir, "model_hparams.json"), "w") as f:
            f.write(json.dumps(model.hparams.values(), sort_keys=True, indent=4))
    model.restore(None, args.checkpoint)

    import cv2
    sample_ind = 0
    while True:
        if args.num_samples and sample_ind >= args.num_samples:
            break
        if sample_ind > 0:
            try:
                inputs = dataset.make_batch(args.batch_size)
            except StopIteration:                     # the reference's tf.errors.OutOfRangeError
                break
        print("evaluation samples from %d to %d" % (sample_ind, sample_ind + args.batch_size))
        for stochastic_sample_ind in range(args.num_stochastic_samples):
            model.global_step = sample_ind * 131 + stochastic_sample_ind     # a fresh noise draw per sess.run
            gen_images = model.predict(inputs)                               # [B, T-1, H, W, C] as outputs['gen_images']
            gen_images = gen_images[:, -future_length:]                      # only keep the future frames
            for i, gen_images_ in enumerate(gen_images):
                context_images_ = (np.asarray(inputs['images'][i]) * 255.0).astype(np.uint8)
                gen_images_ = (gen_images_ * 255.0).astype(np.uint8)
                context_and_gen_images = list(context_images_[:context_frames]) + list(gen_images_)
                if args.gif_length:
                    context_and_gen_images = context_and_gen_images[:args.gif_length]
                stem = os.path.join(args.output_gif_dir, 'gen_image_%05d_%02d' % (sample_ind + i, stochastic_sample_ind))
                np.save(stem + '.npy', np.stack(context_and_gen_images))
                save_gif(stem + '.gif', context_and_gen_images, args.fps)
                pattern = 'gen_image_%%05d_%%02d_%%0%dd.png' % max(2, len(str(len(gen_images_) - 1)))
                for t, gen_image in enumerate(gen_images_):
                    if gen_image.shape[-1] == 1:
                        gen_image = np.tile(gen_image, (1, 1, 3))
                    else:
                        gen_image = cv2.cvtColor(gen_image, cv2.COLOR_RGB2BGR)
                    cv2.imwrite(os.path.join(args.output_png_dir, pattern % (sample_ind + i, stochastic_sample_ind, t)), gen_image)
        sample_ind += args.batch_size
    return sample_ind


if __name__ == '__main__':
    main()
