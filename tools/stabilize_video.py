"""Video stabilisation: the camera's shake removed from a handheld video, its intended motion kept.

    python tools/stabilize_video.py out.mp4 --video_filepath in.mp4 -c weights.params [-n MaskFlownet_S] [--radius 15]
                                    [--crop 0.9] [--batch 8] [--resize 448,1024] [--precision fp32|bf16]

The frames stream through video.VideoStabilizer: the one-direction flow of each consecutive pair and a robust affine fit
of the camera's motion to it (ops.affine_motion) in one CUDA graph per batch, a camera path smoothed over --radius frames
on each side (camera.stabilize_path), and a GPU warp of every frame, zoomed by --crop so that the replicated border stays
mostly out of view.  The output has as many frames as the input, at the input's frame rate (25 when it gives none).
Frames stay in the channel order cv2 reads them (B,G,R); the stabilisation does not depend on it.  -c, -n, --batch,
--resize and --precision are those of predict_new_data.py.
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200.video import VideoStabilizer  # noqa: E402
from predict_new_data import NETWORKS, load_model, open_video, open_video_writer, video_frames  # noqa: E402


@torch.no_grad()
def stabilize_file(model: torch.nn.Module, out_filepath: str, video_filepath: str, radius: int = 15, crop: float = 0.9,
                   batch: int = 8, resize=None):
    """Writes the stabilised video_filepath to out_filepath at the input's frame rate.  Returns (frames written, fps)."""
    cap, fps_in = open_video(video_filepath)
    fps = fps_in if fps_in > 0 else 25.0
    stab = VideoStabilizer(model, batch=batch, resize=resize, radius=radius, crop=crop)
    writer, n = None, 0
    try:
        for fr in stab.run(video_frames(cap)):
            if writer is None:
                writer = open_video_writer(out_filepath, fps, fr.shape)
            writer.write(fr)
            n += 1
    finally:
        if writer is not None:
            writer.release()
    return n, fps


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("out_filepath", help="destination video")
    ap.add_argument("--video_filepath", required=True, help="input video")
    ap.add_argument("-c", "--checkpoint", required=True, help=".params checkpoint or .pt state_dict")
    ap.add_argument("-n", "--network", choices=sorted(NETWORKS), default="MaskFlownet")
    ap.add_argument("--radius", type=int, default=15, help="frames on each side of the camera path's smoothing window")
    ap.add_argument("--crop", type=float, default=0.9, help="zoom about the centre, in (0,1]: the share of the frame shown")
    ap.add_argument("--batch", type=int, default=8, help="frame pairs per graph replay")
    ap.add_argument("--resize", default="", help="network input size H,W (default: the next multiples of 64)")
    ap.add_argument("--precision", choices=("fp32", "bf16"), default="fp32",
                    help="arithmetic of the 3x3 convolutions: fp32-accurate (default) or the faster bf16 mode")
    a = ap.parse_args(argv)
    if a.radius < 0:
        ap.error(f"--radius must be >= 0, got {a.radius}")
    if not 0.0 < a.crop <= 1.0:
        ap.error(f"--crop must lie in (0,1], got {a.crop}")
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
    n, fps = stabilize_file(model, a.out_filepath, a.video_filepath, a.radius, a.crop, a.batch, a.resize)
    print(f"wrote {n} frames at {fps:g} fps to {a.out_filepath}")


if __name__ == "__main__":
    main()
