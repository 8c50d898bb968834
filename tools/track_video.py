"""Dense point tracks through a video: where every textured point (and every query point) goes over the following frames.

    python tools/track_video.py tracks.npz --video_filepath in.mp4 -c weights.params [-n MaskFlownet_S] [--spacing 8]
                                [--queries q.csv] [--overlay out.avi --tail 15] [--batch 8] [--resize 448,1024]
                                [--precision fp32|bf16]

The frames stream through video.VideoTracker: flow in both directions from one feature pyramid, then the tracking steps
(tracks chained along the forward flow, stopped by the forward-backward check or at motion boundaries, reseeded on a
grid of `spacing` pixels where textured cells are uncovered), all in one CUDA graph per batch.  tracks.npz holds
video.collect_tracks' arrays, indexed by track id: start, length, offset, xy (x,y pixels, frame by frame) and reason (0 =
alive in the last frame, 3 = left the frame, 4 = occluded, 5 = motion boundary).  --queries: a CSV file of rows t,x,y
(an optional header line is skipped); query i gets track id i.  --overlay draws each live track's last `tail` positions
on the frames with cv2.  -c, -n, --batch, --resize and --precision are those of predict_new_data.py.
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
from maskflownet_b200.video import VideoTracker, collect_tracks  # noqa: E402
from predict_new_data import add_model_args, model_from_args, parse_model_args, open_video, open_video_writer, video_frames  # noqa: E402


def read_queries(path: str) -> np.ndarray:
    """(M,3) float64 rows (t, x, y) of a CSV file; a first line that is not numeric is a header."""
    rows = []
    with open(path) as f:
        for n, line in enumerate(f):
            line = line.strip()
            if not line:
                continue
            try:
                rows.append([float(v) for v in line.split(",")])
            except ValueError:
                if n == 0:
                    continue
                raise ValueError(f"{path}:{n + 1}: expected t,x,y, got {line!r}") from None
    q = np.asarray(rows, np.float64).reshape(-1, 3) if rows else np.zeros((0, 3))
    return q


def _colour(i: int):
    h = (i * 0.618033988749895) % 1.0
    return tuple(int(255 * (0.5 + 0.5 * np.cos(2 * np.pi * (h + o)))) for o in (0.0, 1 / 3, 2 / 3))


@torch.no_grad()
def track_file(model: torch.nn.Module, out_filepath: str, video_filepath: str, spacing: int = 8, queries=None,
               overlay=None, tail: int = 15, batch: int = 8, resize=None) -> int:
    """Tracks video_filepath and writes collect_tracks' arrays to out_filepath (.npz); with `overlay`, also a copy of the
    video with each live track's last `tail` positions drawn.  Returns the number of frames."""
    cap, fps = open_video(video_filepath)
    tracker = VideoTracker(model, batch=batch, resize=resize, spacing=spacing, queries=queries)
    seen = collections.deque()        # frames read but not yet drawn
    history = {}                      # track id -> its last `tail` positions

    def frames():
        for fr in video_frames(cap):
            if overlay:
                seen.append(fr)
            yield fr

    kept, writer = [], None
    try:
        for tf in tracker.run(frames()):
            kept.append(tf)
            if not overlay:
                continue
            import cv2

            fr = seen.popleft().copy()
            if writer is None:
                writer = open_video_writer(overlay, fps, fr.shape)
            for i in tf.ended_ids:
                history.pop(int(i), None)
            for i, p in zip(tf.ids, tf.xy):
                h = history.setdefault(int(i), collections.deque(maxlen=tail))
                h.append((int(round(float(p[0]))), int(round(float(p[1])))))
                pts = np.asarray(h, np.int32).reshape(-1, 1, 2)
                if len(h) > 1:
                    cv2.polylines(fr, [pts], False, _colour(int(i)), 1, cv2.LINE_AA)
                cv2.circle(fr, h[-1], 1, _colour(int(i)), -1)
            writer.write(fr)
    finally:
        if writer is not None:
            writer.release()
    np.savez(out_filepath, **collect_tracks(kept))
    return len(kept)


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("out_filepath", help="destination .npz of the tracks")
    ap.add_argument("--video_filepath", required=True, help="input video")
    add_model_args(ap)
    ap.add_argument("--spacing", type=int, default=8, help="seeding grid spacing in pixels")
    ap.add_argument("--queries", default=None, help="CSV file of query points t,x,y")
    ap.add_argument("--overlay", default=None, help="also write the video with the tracks drawn")
    ap.add_argument("--tail", type=int, default=15, help="positions drawn per track in the overlay")
    a = parse_model_args(ap, argv)
    try:
        ops.check_track_args(a.spacing, None, "track_video")
    except ops.MaskflowError as e:
        ap.error(str(e))
    if a.tail < 1:
        ap.error(f"--tail must be >= 1, got {a.tail}")
    return a


def main(argv=None):
    a = parse_args(argv)
    model = model_from_args(a)
    q = read_queries(a.queries) if a.queries else None
    n = track_file(model, a.out_filepath, a.video_filepath, a.spacing, q, a.overlay, a.tail, a.batch, a.resize)
    print(f"tracked {n} frames of {a.video_filepath} into {a.out_filepath}")


if __name__ == "__main__":
    main()
