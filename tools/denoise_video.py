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
from predict_new_data import NETWORKS, load_model, open_video, open_video_writer, video_frames  # noqa: E402


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
    ap.add_argument("-c", "--checkpoint", required=True, help=".params checkpoint or .pt state_dict")
    ap.add_argument("-n", "--network", choices=sorted(NETWORKS), default="MaskFlownet")
    ap.add_argument("--radius", type=int, default=ops.DENOISE_RADIUS, help="neighbouring frames averaged on each side")
    ap.add_argument("--sigma", type=float, default=None,
                    help="noise level in grey levels (default: estimated from the first frames)")
    ap.add_argument("--h", type=float, default=ops.DENOISE_H, help="weight scale, in units of the noise level")
    ap.add_argument("--patch", type=int, default=ops.DENOISE_PATCH,
                    help=f"patch radius of the weights, in [0,{ops.DENOISE_MAX_PATCH}]")
    ap.add_argument("--batch", type=int, default=8, help="frame pairs per graph replay")
    ap.add_argument("--resize", default="", help="network input size H,W (default: the next multiples of 64)")
    ap.add_argument("--precision", choices=("fp32", "bf16"), default="fp32",
                    help="arithmetic of the 3x3 convolutions: fp32-accurate (default) or the faster bf16 mode")
    a = ap.parse_args(argv)
    if a.radius < 0:
        ap.error(f"--radius must be >= 0, got {a.radius}")
    if a.sigma is not None and not 0.0 < a.sigma < float("inf"):
        ap.error(f"--sigma must be positive and finite, got {a.sigma}")
    if not 0.0 < a.h < float("inf"):
        ap.error(f"--h must be positive and finite, got {a.h}")
    if not 0 <= a.patch <= ops.DENOISE_MAX_PATCH:
        ap.error(f"--patch must lie in [0,{ops.DENOISE_MAX_PATCH}], got {a.patch}")
    if a.batch < 1:
        ap.error(f"--batch must be >= 1, got {a.batch}")
    try:
        a.resize = tuple(int(s) for s in a.resize.split(",")) if a.resize else None
    except ValueError:
        ap.error(f"--resize takes H,W, got {a.resize!r}")
    if a.resize is not None and len(a.resize) != 2:
        ap.error(f"--resize takes H,W, got {a.resize}")
    return a


def main(argv=None):
    a = parse_args(argv)
    model = load_model(a.network, a.checkpoint)
    model.inference_precision = a.precision
    n, fps, sigma = denoise_file(model, a.out_filepath, a.video_filepath, a.radius, a.sigma, a.h, a.patch, a.batch,
                                 a.resize)
    print(f"wrote {n} frames at {fps:g} fps to {a.out_filepath} (noise level {sigma:.2f} grey levels)")


if __name__ == "__main__":
    main()
