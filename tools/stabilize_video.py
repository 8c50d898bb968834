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
from maskflownet_b200 import MaskflowError, camera  # noqa: E402
from maskflownet_b200.video import VideoStabilizer  # noqa: E402
from predict_new_data import add_model_args, model_from_args, parse_model_args, open_video, open_video_writer, video_frames  # noqa: E402


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
    add_model_args(ap)
    ap.add_argument("--radius", type=int, default=15, help="frames on each side of the camera path's smoothing window")
    ap.add_argument("--crop", type=float, default=0.9, help="zoom about the centre, in (0,1]: the share of the frame shown")
    a = parse_model_args(ap, argv)
    try:
        camera.check_path_args(a.radius, a.crop, "stabilize_video")
    except MaskflowError as e:
        ap.error(str(e))
    return a


def main(argv=None):
    a = parse_args(argv)
    model = model_from_args(a)
    n, fps = stabilize_file(model, a.out_filepath, a.video_filepath, a.radius, a.crop, a.batch, a.resize)
    print(f"wrote {n} frames at {fps:g} fps to {a.out_filepath}")


if __name__ == "__main__":
    main()
