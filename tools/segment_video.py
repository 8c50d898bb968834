"""Moving-object segmentation of a video: in every frame, the objects that move relative to the camera.

    python tools/segment_video.py objects.npz --video_filepath in.mp4 -c weights.params [-n MaskFlownet_S]
                                  [--tau-lo 1.0] [--tau-hi 2.0] [--min-area 64] [--overlay out.avi] [--batch 8]
                                  [--resize 448,1024] [--precision fp32|bf16]

The frames stream through video.VideoMotionSegmenter: flow in both directions from one feature pyramid, the occlusion
masks, one robust affine camera fit per direction and pair, and the segmentation of each frame from the camera-relative
motion of both directions (ops.segment_motion states the rule), all in one CUDA graph per batch.  objects.npz holds
"labels" (T,H,W) uint8 (object k at the pixels labelled k, 0 elsewhere), "objects" (sum(count),10) float64 rows of
"columns" (area, x0, y0, x1, y1, cx, cy, peak, dx, dy), frame t's rows starting at "offset"[t], "count" (T,) and
"dropped" (T,), the objects past 255.  Objects are numbered per frame; they carry no identity from frame to frame.
--overlay writes the frames with each object tinted and boxed, drawn with cv2.  -c, -n, --batch, --resize and
--precision are those of predict_new_data.py.
"""
from __future__ import annotations

import argparse
import collections
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import ops  # noqa: E402
from maskflownet_b200.video import VideoMotionSegmenter  # noqa: E402
from predict_new_data import add_model_args, model_from_args, parse_model_args, open_video, open_video_writer, video_frames  # noqa: E402

COLUMNS = ("area", "x0", "y0", "x1", "y1", "cx", "cy", "peak", "dx", "dy")


def pack_frames(frames) -> dict:
    """The arrays of objects.npz from a sequence of MotionFrames."""
    frames = list(frames)
    count = np.array([len(f.objects) for f in frames], np.int64)
    rows = [np.asarray(f.objects, np.float64).reshape(-1, 10) for f in frames]
    return {"labels": np.stack([f.labels for f in frames]) if frames else np.zeros((0, 0, 0), np.uint8),
            "objects": np.concatenate(rows) if rows else np.zeros((0, 10)), "count": count,
            "offset": np.cumsum(count) - count, "dropped": np.array([f.dropped for f in frames], np.int64),
            "columns": np.array(COLUMNS)}


def _colour(i: int):
    h = (i * 0.618033988749895) % 1.0
    return tuple(int(255 * (0.5 + 0.5 * np.cos(2 * np.pi * (h + o)))) for o in (0.0, 1 / 3, 2 / 3))


def draw(frame: np.ndarray, mf) -> np.ndarray:
    """frame with each object of the MotionFrame tinted half-way to its colour and boxed."""
    import cv2

    out = frame.copy()
    for k, row in enumerate(mf.objects):
        c = np.array(_colour(k), np.float64)
        m = mf.labels == k + 1
        out[m] = np.rint(0.5 * out[m] + 0.5 * c).astype(np.uint8)
        x0, y0, x1, y1 = (int(v) for v in row[1:5])
        cv2.rectangle(out, (x0, y0), (x1, y1), _colour(k), 1)
    return out


@torch.no_grad()
def segment_file(model: torch.nn.Module, out_filepath: str, video_filepath: str, tau_lo: float = ops.SEG_TAU_LO,
                 tau_hi: float = ops.SEG_TAU_HI, min_area: int = ops.SEG_MIN_AREA, overlay=None, batch: int = 8,
                 resize=None) -> int:
    """Segments video_filepath and writes pack_frames' arrays to out_filepath (.npz); with `overlay`, also a copy of the
    video with the objects drawn.  Returns the number of frames."""
    cap, fps = open_video(video_filepath)
    seg = VideoMotionSegmenter(model, batch=batch, resize=resize, tau_lo=tau_lo, tau_hi=tau_hi, min_area=min_area)
    seen = collections.deque()        # frames read but not yet drawn

    def frames():
        for fr in video_frames(cap):
            if overlay:
                seen.append(fr)
            yield fr

    kept, writer = [], None
    try:
        for mf in seg.run(frames()):
            kept.append(mf)
            if not overlay:
                continue
            fr = seen.popleft()
            if writer is None:
                writer = open_video_writer(overlay, fps, fr.shape)
            writer.write(draw(fr, mf))
    finally:
        if writer is not None:
            writer.release()
    np.savez(out_filepath, **pack_frames(kept))
    return len(kept)


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("out_filepath", help="destination .npz of the objects")
    ap.add_argument("--video_filepath", required=True, help="input video")
    add_model_args(ap)
    ap.add_argument("--tau-lo", type=float, default=ops.SEG_TAU_LO,
                    help="pixels moving at least this far (px) relative to the camera may belong to an object")
    ap.add_argument("--tau-hi", type=float, default=ops.SEG_TAU_HI,
                    help="an object has at least one pixel moving this far (px) relative to the camera")
    ap.add_argument("--min-area", type=int, default=ops.SEG_MIN_AREA, help="smallest object in pixels")
    ap.add_argument("--overlay", default=None, help="also write the video with the objects drawn")
    a = parse_model_args(ap, argv)
    try:
        ops.check_segment_args(a.tau_lo, a.tau_hi, a.min_area, ops.SEG_MAX_OBJECTS, "segment_video")
    except ops.MaskflowError as e:
        ap.error(str(e))
    return a


def main(argv=None):
    a = parse_args(argv)
    model = model_from_args(a)
    n = segment_file(model, a.out_filepath, a.video_filepath, a.tau_lo, a.tau_hi, a.min_area, a.overlay, a.batch,
                     a.resize)
    print(f"segmented {n} frames of {a.video_filepath} into {a.out_filepath}")


if __name__ == "__main__":
    main()
