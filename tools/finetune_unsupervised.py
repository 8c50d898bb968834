"""Fine-tune a flow checkpoint on a user's own unlabelled footage: no flow labels, the unsupervised losses of UnFlow
(Meister, Hur and Roth, AAAI 2018) through PipelineFlownet.train_batch_unsupervised.

    python tools/finetune_unsupervised.py --video_filepath in.mp4 -c weights.params -o tuned [-n MaskFlownet_S]
                                          [--crop 384x512] [--batch 4] [--steps 1000] [--lr 1e-5] [--color-aug]
                                          [--smooth-weight W] [--deterministic] [--seed 0]
    python tools/finetune_unsupervised.py --frames_dir frames/ -c weights.params -o tuned ...

Frames are read with cv2, converted from its B,G,R to R,G,B (the order the census grey weights assume), and kept on
the host.  Every step takes
--batch random pairs of consecutive frames and one random --crop (multiples of 64) per pair, the same window in both
frames.  The result is written with PipelineFlownet.save as PREFIX.pt (the network's state dict, which
`predict_new_data.py -c PREFIX.pt` loads) and PREFIX.states.pt (Adam's state).
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

NETWORKS = ("MaskFlownet", "MaskFlownet_S")
IMAGE_EXT = (".png", ".jpg", ".jpeg", ".bmp", ".ppm", ".tif", ".tiff")


def _crop(text: str):
    try:
        h, w = (int(v) for v in text.lower().split("x"))
    except ValueError:
        raise argparse.ArgumentTypeError(f"--crop takes HxW, got {text!r}")
    if h <= 0 or w <= 0 or h % 64 or w % 64:
        raise argparse.ArgumentTypeError(f"--crop: H and W must be positive multiples of 64, got {text!r}")
    return h, w


def _positive(text: str):
    v = int(text)
    if v <= 0:
        raise argparse.ArgumentTypeError(f"expected a positive integer, got {text!r}")
    return v


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--video_filepath", help="input video")
    src.add_argument("--frames_dir", help="directory of frames, taken in file-name order")
    ap.add_argument("-c", "--checkpoint", required=True, help=".params checkpoint or .pt state_dict to start from")
    ap.add_argument("-n", "--network", choices=NETWORKS, default="MaskFlownet_S")
    ap.add_argument("-o", "--output", required=True, metavar="PREFIX", help="writes PREFIX.pt and PREFIX.states.pt")
    ap.add_argument("--crop", type=_crop, default=(384, 512), help="training crop HxW, multiples of 64 (default 384x512)")
    ap.add_argument("--batch", type=_positive, default=4, help="frame pairs per step")
    ap.add_argument("--steps", type=_positive, default=1000)
    ap.add_argument("--lr", type=float, default=1e-5, help="Adam learning rate")
    ap.add_argument("--color-aug", action="store_true", help="colour augmentation of the network input")
    ap.add_argument("--smooth-weight", type=float, default=None, help="weight of the smoothness term (default: the "
                                                                         "pipeline's SMOOTH_WEIGHT)")
    ap.add_argument("--deterministic", action="store_true", help="bit-reproducible steps (PipelineFlownet deterministic)")
    ap.add_argument("--seed", type=int, default=0, help="seed of the pair / crop sampling, the colour augmentation and "
                                                        "torch")
    return ap.parse_args(argv)


def read_frames(video_filepath=None, frames_dir=None):
    """All frames as (H,W,3) uint8 R,G,B arrays on the host."""
    import cv2
    frames = []
    if video_filepath is not None:
        cap = cv2.VideoCapture(video_filepath)
        if not cap.isOpened():
            raise FileNotFoundError(f"cannot open video {video_filepath}")
        try:
            while True:
                ok, frame = cap.read()
                if not ok:
                    break
                frames.append(np.ascontiguousarray(frame[..., ::-1]))
        finally:
            cap.release()
    else:
        names = sorted(f for f in os.listdir(frames_dir) if f.lower().endswith(IMAGE_EXT))
        for name in names:
            frame = cv2.imread(os.path.join(frames_dir, name))
            if frame is None:
                raise FileNotFoundError(f"cannot read image {os.path.join(frames_dir, name)}")
            frames.append(np.ascontiguousarray(frame[..., ::-1]))
    if frames and any(f.shape != frames[0].shape for f in frames):
        raise ValueError("the frames differ in size")
    return frames


def sample_batch(frames, batch: int, crop, rng):
    """(img1, img2) (batch,3,h,w) uint8: random consecutive pairs, one random crop per pair; and (idx, ys, xs)."""
    if len(frames) < 2:
        raise ValueError("fine-tuning needs at least two frames")
    H, W = frames[0].shape[:2]
    h, w = crop
    if h > H or w > W:
        raise ValueError(f"the crop {h}x{w} is larger than the frames ({H}x{W})")
    idx = rng.integers(0, len(frames) - 1, batch)
    ys, xs = rng.integers(0, H - h + 1, batch), rng.integers(0, W - w + 1, batch)
    img1 = np.stack([frames[i][y:y + h, x:x + w] for i, y, x in zip(idx, ys, xs)]).transpose(0, 3, 1, 2)
    img2 = np.stack([frames[i + 1][y:y + h, x:x + w] for i, y, x in zip(idx, ys, xs)]).transpose(0, 3, 1, 2)
    return np.ascontiguousarray(img1), np.ascontiguousarray(img2), (idx, ys, xs)


def color_augmentation(batch: int, crop, seed: int):
    """The colour augmentation of the reference's Sintel fine-tuning configuration (main.py), for the network input
    only."""
    from maskflownet_b200.augment import ColorAugmentation
    return ColorAugmentation(contrast_range=(-0.4, 0.8), brightness_sigma=0.1, channel_range=(0.8, 1.4),
                             batch_size=batch, shape=tuple(crop), noise_range=(0, 0), saturation=0.5, hue=0.5,
                             eigen_aug=False, seed=seed)


def finetune(a, log=print):
    import torch
    from maskflownet_b200 import pipeline

    torch.manual_seed(a.seed)
    frames = read_frames(a.video_filepath, a.frames_dir)
    kw = {} if a.smooth_weight is None else {"smooth_weight": a.smooth_weight}
    pipe = pipeline.PipelineFlownet(network_class=a.network, learning_rate=a.lr, deterministic=a.deterministic, **kw)
    pipe.load(a.checkpoint)
    aug = color_augmentation(a.batch, a.crop, a.seed) if a.color_aug else None
    rng = np.random.default_rng(a.seed)
    t0, hist = time.time(), []
    for step in range(1, a.steps + 1):
        img1, img2, _ = sample_batch(frames, a.batch, a.crop, rng)
        out = pipe.train_batch_unsupervised(img1, img2, color_aug=aug)
        hist.append(out)
        if step == 1 or step % 50 == 0 or step == a.steps:
            log(f"step {step}/{a.steps}: loss {out['loss']:.4f} (census {out['photo']:.4f}, smoothness "
                f"{out['smooth']:.4f}), occluded {100 * out['occluded']:.1f} %, {time.time() - t0:.0f} s")
    pipe.save(a.output)
    log(f"wrote {a.output}.pt and {a.output}.states.pt")
    return hist


def main(argv=None):
    finetune(parse_args(argv))


if __name__ == "__main__":
    main()
