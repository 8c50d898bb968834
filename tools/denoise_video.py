"""Video denoising: each frame averaged with its neighbours aligned along the flow, weighted so a wrong flow cannot ghost.

    python tools/denoise_video.py out.mp4 --video_filepath in.mp4 -c weights.params [-n MaskFlownet_S] [--radius 2]
                                  [--sigma 10] [--h 0.7] [--patch 1] [--batch 8] [--resize 448,1024]
                                  [--precision fp32|bf16]

The frames stream through video.VideoDenoiser: both flow directions of each consecutive pair in one CUDA graph per
batch, then on the GPU each frame is averaged with up to --radius neighbours on each side, aligned along the chained
flow and weighted by the colour distance of a (2 --patch + 1)^2 patch against h = --h times the noise level
(ops.denoise_frames).  --sigma is the noise level in grey levels; without it, it is estimated from the first frames
(ops.median_noise).  The output has as many frames as the input, at the input's frame rate (25 when it gives none).
Frames stay in the channel order cv2 reads them (B,G,R); the denoising does not depend on it.  -c, -n, --batch, --resize
and --precision are those of predict_new_data.py.
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import ops  # noqa: E402
from maskflownet_b200.video import VideoDenoiser  # noqa: E402
from predict_new_data import add_model_args, model_from_args, parse_model_args, open_video, open_video_writer, video_frames  # noqa: E402


@torch.no_grad()
def denoise_file(model: torch.nn.Module, out_filepath: str, video_filepath: str, radius: int = ops.DENOISE_RADIUS,
                 sigma=None, h: float = ops.DENOISE_H, patch: int = ops.DENOISE_PATCH, batch: int = 8, resize=None):
    """Writes the denoised video_filepath to out_filepath at the input's frame rate.  Returns (frames written, fps,
    the noise level used)."""
    cap, fps_in = open_video(video_filepath)
    fps = fps_in if fps_in > 0 else 25.0
    den = VideoDenoiser(model, batch=batch, resize=resize, radius=radius, sigma=sigma, h=h, patch=patch)
    writer, n = None, 0
    try:
        for fr in den.run(video_frames(cap)):
            if writer is None:
                writer = open_video_writer(out_filepath, fps, fr.shape)
            writer.write(fr)
            n += 1
    finally:
        if writer is not None:
            writer.release()
    return n, fps, den.sigma_used


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("out_filepath", help="destination video")
    ap.add_argument("--video_filepath", required=True, help="input video")
    add_model_args(ap)
    ap.add_argument("--radius", type=int, default=ops.DENOISE_RADIUS, help="neighbouring frames averaged on each side")
    ap.add_argument("--sigma", type=float, default=None,
                    help="noise level in grey levels (default: estimated from the first frames)")
    ap.add_argument("--h", type=float, default=ops.DENOISE_H, help="weight scale, in units of the noise level")
    ap.add_argument("--patch", type=int, default=ops.DENOISE_PATCH,
                    help=f"patch radius of the weights, in [0,{ops.DENOISE_MAX_PATCH}]")
    a = parse_model_args(ap, argv)
    try:
        ops.check_denoise_args(a.radius, a.sigma, a.h, a.patch, 0.01, 0.5, "denoise_video", sigma_optional=True)
    except ops.MaskflowError as e:
        ap.error(str(e))
    return a


def main(argv=None):
    a = parse_args(argv)
    model = model_from_args(a)
    n, fps, sigma = denoise_file(model, a.out_filepath, a.video_filepath, a.radius, a.sigma, a.h, a.patch, a.batch,
                                 a.resize)
    print(f"wrote {n} frames at {fps:g} fps to {a.out_filepath} (noise level {sigma:.2f} grey levels)")


if __name__ == "__main__":
    main()
