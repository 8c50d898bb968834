"""Flow of a user's own data, written as the Middlebury colour coding: the reference's predict_new_data.py on this library.

    python tools/predict_new_data.py out.png --image_1 a.png --image_2 b.png -c weights.params [-n MaskFlownet_S]
    python tools/predict_new_data.py out.avi --video_filepath in.mp4 -c weights.params [--batch 8] [--resize 448,1024]
                                     [--max_radius 20] [--occlusion occ.avi]

An image pair gives one PNG.  A video gives a video of the input's frame rate with one colour frame per consecutive frame
pair (so one frame fewer than the input), streamed through network.VideoFlowPredictor: each frame is uploaded once and
coloured on the GPU.  Frames go to the network in the channel order cv2 reads them (B,G,R), as in the reference.

-c takes a shipped .params checkpoint (maskflownet_b200.params.load_checkpoint) or a .pt state_dict of the model class
-n names.  Departures from the reference, on purpose:
  * the PNG has standard colours.  The reference hands an RGB image to cv2.imwrite, which expects B,G,R, so its PNGs have
    red and blue swapped; here the colour kernel writes B,G,R for cv2.
  * --resize is honoured.  The reference parses it but passes it to neither the image nor the video path.
  * videos are written with cv2.VideoWriter (MJPG for .avi, mp4v otherwise) instead of moviepy; there is no audio.
  * --max_radius (new) fixes the colour scale across frames; by default every frame is normalised by its own largest
    flow, as flow_vis does.
  * --occlusion PATH (new) also writes the forward-backward occlusion mask of each pair's first image (255 = occluded:
    no consistent match in the second image, ops.flow_consistency): an 8-bit image for a pair, a greyscale video of one
    frame per pair for a video.  The pair is then predicted in both directions from one feature pyramid
    (network.predict_bidirectional); the flow written is the forward one of that run.
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import network, ops, params  # noqa: E402
from maskflownet_b200.video import VideoFlowPredictor  # noqa: E402

NETWORKS = {"MaskFlownet": network.MaskFlownet, "MaskFlownet_S": network.MaskFlownetS}


def load_model(name: str, checkpoint: str, device="cuda") -> torch.nn.Module:
    model = NETWORKS[name]()
    if checkpoint.endswith(".params"):
        params.load_checkpoint(model, checkpoint)
    else:
        model.load_state_dict(torch.load(checkpoint, map_location="cpu"))
    return model.to(device).eval()


def add_model_args(ap: argparse.ArgumentParser) -> None:
    """The options every tool shares: -c/-n (the model), --batch, --resize and --precision.  parse_model_args checks
    them and model_from_args loads the model they name."""
    ap.add_argument("-c", "--checkpoint", required=True, help=".params checkpoint or .pt state_dict")
    ap.add_argument("-n", "--network", choices=sorted(NETWORKS), default="MaskFlownet")
    ap.add_argument("--batch", type=int, default=8, help="frame pairs per graph replay")
    ap.add_argument("--resize", default="", help="network input size H,W (default: the next multiples of 64)")
    ap.add_argument("--precision", choices=("fp32", "bf16"), default="fp32",
                    help="arithmetic of the 3x3 convolutions: fp32-accurate (default) or the faster bf16 mode")


def parse_model_args(ap: argparse.ArgumentParser, argv=None) -> argparse.Namespace:
    """ap.parse_args(argv) with --batch checked and --resize turned into (H, W) (None when not given)."""
    a = ap.parse_args(argv)
    if a.batch < 1:
        ap.error(f"--batch must be >= 1, got {a.batch}")
    try:
        a.resize = tuple(int(s) for s in a.resize.split(",")) if a.resize else None
    except ValueError:
        ap.error(f"--resize takes H,W, got {a.resize!r}")
    if a.resize is not None and len(a.resize) != 2:
        ap.error(f"--resize takes H,W, got {a.resize}")
    return a


def model_from_args(a: argparse.Namespace) -> torch.nn.Module:
    """The model of -c/-n on the GPU, at the arithmetic of --precision."""
    model = load_model(a.network, a.checkpoint)
    model.inference_precision = a.precision
    return model


def open_video(path: str):
    """(cv2.VideoCapture, frame rate) of a video file; the rate is 0 when the container does not give one."""
    import cv2

    cap = cv2.VideoCapture(path)
    if not cap.isOpened():
        raise FileNotFoundError(f"cannot open video {path}")
    return cap, cap.get(cv2.CAP_PROP_FPS)


def video_frames(cap):
    """The frames of an open cv2.VideoCapture (H,W,3) uint8 B,G,R, in order; releases it at the end."""
    try:
        while True:
            ok, frame = cap.read()
            if not ok:
                return
            yield frame
    finally:
        cap.release()


def open_video_writer(path: str, fps: float, shape):
    """cv2.VideoWriter of (H,W,...) frames at `fps` (25 when fps is not positive): MJPG for .avi, mp4v otherwise."""
    import cv2

    fourcc = cv2.VideoWriter_fourcc(*("MJPG" if path.lower().endswith(".avi") else "mp4v"))
    w = cv2.VideoWriter(path, fourcc, fps if fps > 0 else 25.0, (shape[1], shape[0]))
    if not w.isOpened():
        raise OSError(f"cannot write {path}")
    return w


def _imread(cv2, path):
    img = cv2.imread(path)
    if img is None:
        raise FileNotFoundError(f"cannot read image {path}")
    return img


@torch.no_grad()
def predict_files(model: torch.nn.Module, flow_filepath: str, image_1=None, image_2=None, video_filepath=None, batch=8,
                  resize=None, max_radius=None, occlusion_filepath=None) -> int:
    """Writes the colour-coded flow of an image pair (one image) or of a video (one frame per consecutive pair) to
    flow_filepath, and with occlusion_filepath the occlusion masks of the pairs' first images there (255 = occluded);
    returns the number of flow images written."""
    import cv2

    if video_filepath is None:
        if image_1 is None or image_2 is None:
            raise ValueError("give --image_1 and --image_2, or --video_filepath")
        a, b = _imread(cv2, image_1), _imread(cv2, image_2)
        if a.shape != b.shape:
            raise ValueError(f"the images differ in size: {a.shape} vs {b.shape}")
        dev = next(model.parameters()).device
        to_dev = lambda im: torch.from_numpy(im).permute(2, 0, 1)[None].contiguous().to(dev)  # noqa: E731
        if occlusion_filepath is None:
            flow, _ = network.predict(model, to_dev(a), to_dev(b), resize)
        else:
            flow, _, occ, _ = network.predict_bidirectional(model, to_dev(a), to_dev(b), resize)
            if not cv2.imwrite(occlusion_filepath, (occ[0] * 255).cpu().numpy()):
                raise OSError(f"cannot write {occlusion_filepath}")
        rgb, _ = ops.flow_to_color(flow[0], max_radius, bgr=True)
        if not cv2.imwrite(flow_filepath, rgb.cpu().numpy()):
            raise OSError(f"cannot write {flow_filepath}")
        return 1

    cap, fps = open_video(video_filepath)
    bidirectional = occlusion_filepath is not None
    pred = VideoFlowPredictor(model, batch=batch, resize=resize, max_radius=max_radius, bgr=True,
                              bidirectional=bidirectional)

    writers, n = [], 0
    try:
        for res in pred.run(video_frames(cap)):
            rgb = res[0] if bidirectional else res
            if not writers:
                writers.append(open_video_writer(flow_filepath, fps, rgb.shape))
                if bidirectional:
                    writers.append(open_video_writer(occlusion_filepath, fps, rgb.shape))
            writers[0].write(rgb)
            if bidirectional:   # grey frames through the colour writer: 255 = occluded in all three channels
                writers[1].write(cv2.cvtColor(res[1] * 255, cv2.COLOR_GRAY2BGR))
            n += 1
    finally:
        for w in writers:
            w.release()
    return n


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("flow_filepath", help="destination of the flow image / video")
    ap.add_argument("--image_1", help="first image")
    ap.add_argument("--image_2", help="second image")
    ap.add_argument("--video_filepath", help="input video")
    add_model_args(ap)
    ap.add_argument("--max_radius", type=float, default=None,
                    help="fixed flow magnitude (pixels) of the colour wheel's rim; default: each frame's largest flow")
    ap.add_argument("--occlusion", default=None, metavar="PATH",
                    help="also write the forward-backward occlusion mask of each pair (255 = occluded) to PATH: an image "
                         "for an image pair, a video for a video")
    a = parse_model_args(ap, argv)
    if a.video_filepath is None and (a.image_1 is None or a.image_2 is None):
        ap.error("give --image_1 and --image_2, or --video_filepath")
    n = predict_files(model_from_args(a), a.flow_filepath, a.image_1, a.image_2, a.video_filepath, a.batch, a.resize,
                      a.max_radius, a.occlusion)
    print(f"wrote {n} image(s) to {a.flow_filepath}" + (f" and their occlusion masks to {a.occlusion}" if a.occlusion else ""))


if __name__ == "__main__":
    main()
