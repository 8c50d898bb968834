"""Frame-rate up-conversion and slow motion: F-1 in-between frames for every consecutive frame pair of a video.

    python tools/interpolate_video.py out.mp4 --video_filepath in.mp4 -c weights.params [-n MaskFlownet_S] --factor F
                                      [--batch 8] [--resize 448,1024] [--precision fp32|bf16] [--fps R]

The pairs stream through network.VideoFlowPredictor(interpolate=F-1): flow in both directions from one feature pyramid,
the forward-backward occlusion masks and occlusion-weighted forward splatting of both frames (ops.interpolate_frames), all
in one CUDA graph per batch, at the times k / F, k = 1..F-1.  The output holds frame 0, then for each pair its F-1
in-between frames and the pair's second frame: (n-1) F + 1 frames for n input frames.  Its frame rate is the input's
times F (frame-rate up-conversion, e.g. 30 -> 60 fps with --factor 2); --fps sets it, e.g. to the input's rate for
F-times slow motion.  Frames stay in the channel order cv2 reads them (B,G,R); the interpolation does not depend on it.
-c, -n, --batch, --resize and --precision are those of predict_new_data.py.
"""
from __future__ import annotations

import argparse
import collections
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200.video import VideoFlowPredictor  # noqa: E402
from predict_new_data import add_model_args, model_from_args, parse_model_args, open_video, open_video_writer, video_frames  # noqa: E402


@torch.no_grad()
def interpolate_file(model: torch.nn.Module, out_filepath: str, video_filepath: str, factor: int, batch: int = 8,
                     resize=None, fps=None):
    """Writes video_filepath with factor-1 interpolated frames between consecutive frames to out_filepath, at `fps`
    (default: the input's rate times factor; 25 times factor when the input gives none).  Returns (frames written, fps)."""
    if factor < 2:
        raise ValueError(f"factor must be >= 2, got {factor}")
    cap, fps_in = open_video(video_filepath)
    fps_out = float(fps) if fps is not None else (fps_in if fps_in > 0 else 25.0) * factor
    pred = VideoFlowPredictor(model, batch=batch, resize=resize, interpolate=factor - 1)
    seen = collections.deque()        # input frames read but not yet written: frame t and t+1 of the next result

    def frames():
        for fr in video_frames(cap):
            seen.append(fr)
            yield fr

    writer, n = None, 0
    try:
        for stack in pred.run(frames()):
            if writer is None:
                writer = open_video_writer(out_filepath, fps_out, stack.shape[1:])
                writer.write(seen[0])
                n += 1
            seen.popleft()
            for fr in stack:
                writer.write(fr)
            writer.write(seen[0])
            n += len(stack) + 1
        if writer is None and seen:   # a one-frame video: nothing to interpolate
            writer = open_video_writer(out_filepath, fps_out, seen[0].shape)
            writer.write(seen[0])
            n = 1
    finally:
        if writer is not None:
            writer.release()
    return n, fps_out


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("out_filepath", help="destination video")
    ap.add_argument("--video_filepath", required=True, help="input video")
    add_model_args(ap)
    ap.add_argument("--factor", type=int, required=True, help="F >= 2: F-1 new frames between consecutive input frames")
    ap.add_argument("--fps", type=float, default=None,
                    help="output frame rate (default: the input's times F; the input's own rate gives slow motion)")
    a = parse_model_args(ap, argv)
    if a.factor < 2:
        ap.error(f"--factor must be >= 2, got {a.factor}")
    if a.fps is not None and not 0.0 < a.fps < float("inf"):
        ap.error(f"--fps must be positive, got {a.fps}")
    return a


def main(argv=None):
    a = parse_args(argv)
    model = model_from_args(a)
    n, fps = interpolate_file(model, a.out_filepath, a.video_filepath, a.factor, a.batch, a.resize, a.fps)
    print(f"wrote {n} frames at {fps:g} fps to {a.out_filepath}")


if __name__ == "__main__":
    main()
