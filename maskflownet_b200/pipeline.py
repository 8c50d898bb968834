"""Host-side mirror of the reference's `PipelineFlownet` (/root/reference/network/pipeline.py:19-223): the class `main.py`
drives -- same method names, argument meaning and return values -- composed from this package's operators:

    train_batch   pipeline.py:89-115   /255, geo_aug, color_aug (augment.py), centralize, network (tensor-core forward under
                                       autograd), labels.flip, MultiscaleEpe (fused), backward, ONE gradient all-reduce,
                                       Adam step rescaled by 1/batch_size (Trainer.step(batch_size)), EPE metric
    train_batch_unsupervised           (not in the reference) the same step on unlabelled pairs: network at batch 2n on
                                       both directions, losses.unsupervised_loss (census + smoothness, occlusion-masked)
    do_batch_mx   pipeline.py:117-132  centralize + BilinearResize2D to multiples of 64 (ops.preprocess) + network
    do_batch      pipeline.py:134-147  Upsample(4), resize back + per-channel rescale, Reconstruction2DSmooth, masked EPE
    validate      pipeline.py:149-187  dataset loop -> mean EPE, or the KITTI outlier ratio (return_type != 'epe')
    predict       pipeline.py:189-223  dataset loop -> (flow (H,W,2) in (x,y), occlusion mask, warped image) per sample
    set_learning_rate / lr / save / load / load_head / fix_head    pipeline.py:52-79

One process drives ONE GPU (the reference splits a batch over a context list inside the process; here the launcher starts
one rank per GPU and `train_batch` receives this rank's shard -- dist.shard_batch -- the all-reduce does the rest).
Images arrive as uint8 NCHW arrays / tensors like the reference's (`img / 255.0` happens on the device).
"""
from __future__ import annotations

import contextlib
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import dist as mdist
from . import losses, network, ops, params as mparams
from ._lib import MaskflowError

STRIDES = (64, 32, 16, 8, 4)
SMOOTH_WEIGHT = 3.0     # train_batch_unsupervised's weight of the smoothness term (README, "Unsupervised fine-tuning")


def _to_device(x, device, dtype=None) -> torch.Tensor:
    t = torch.from_numpy(np.ascontiguousarray(x)) if isinstance(x, np.ndarray) else x
    t = t.to(device, non_blocking=True)
    return t if dtype is None else t.to(dtype)


def epe_loss_with_mask(pred: torch.Tensor, label: torch.Tensor, mask: torch.Tensor, eps: float = 1e-8) -> torch.Tensor:
    """EpeLossWithMask (network/MaskFlownet.py:563-583): per-sample masked mean end-point error."""
    return losses.epe_loss_with_mask(pred, label, mask, eps)


class PipelineFlownet:
    """deterministic=True makes train_batch, do_batch(_mx), validate and predict bit-reproducible: each call runs under
    torch.use_deterministic_algorithms(True) (restored afterwards), so this library's ops take their *_det kernels and torch
    picks deterministic cuDNN algorithms.  torch.backends.cudnn.benchmark must stay off (it may pick a different algorithm
    per run; the pipeline raises if it is on), and the process must be started with CUBLAS_WORKSPACE_CONFIG=:4096:8 (or
    :16:8) in the environment, which torch requires for deterministic cuBLAS calls.
    precision: the network's inference_precision ("fp32" or the opt-in "bf16") for do_batch_mx, do_batch, validate and
    predict; train_batch always trains with fp32-accurate arithmetic."""
    _lr = None

    def __init__(self, device=None, network_class: str = "MaskFlownet_S", lr_schedule: Optional[Sequence[Tuple[int, float]]] = None,
                 multiscale_weights: Sequence[float] = losses.WEIGHTS, q: Optional[float] = None, learning_rate: float = 1e-4,
                 deterministic: bool = False, precision: str = "fp32", smooth_weight: float = SMOOTH_WEIGHT):
        if precision not in network.PRECISIONS:
            raise MaskflowError(f"PipelineFlownet: precision must be one of {network.PRECISIONS}, got {precision!r}")
        self.precision = precision
        self.deterministic = bool(deterministic)
        self._check_deterministic_settings()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        cls = {"MaskFlownet_S": network.MaskFlownetS, "MaskFlownet": network.MaskFlownet}.get(network_class)
        if cls is None:
            raise MaskflowError(f"PipelineFlownet: unknown network class {network_class!r} (MaskFlownet_S | MaskFlownet)")
        self.network = cls().to(self.device)                       # MSRAPrelu(slope=0.1) initialisation (pipeline.py:26)
        if precision != "fp32":
            self.network.inference_precision = precision
        self.trainer = torch.optim.Adam(self.network.parameters(), lr=learning_rate)      # gluon.Trainer 'adam' 1e-4 (:27)
        self._lr = learning_rate
        self.strides = list(STRIDES)
        self.scale = self.strides[-1]
        w = list(multiscale_weights)
        self.multiscale_weights = w if len(w) == 5 else list(losses.WEIGHTS)              # pipeline.py:39-41
        self.q = q
        self.lr_schedule = list(lr_schedule) if lr_schedule is not None else []
        self.smooth_weight = float(smooth_weight)
        self._bucket: Optional[mdist.GradBucket] = None

    # ---- deterministic mode -------------------------------------------------------------------------------------
    def _check_deterministic_settings(self) -> None:
        if self.deterministic and torch.backends.cudnn.benchmark:
            raise MaskflowError("PipelineFlownet(deterministic=True): torch.backends.cudnn.benchmark is on; benchmark mode "
                                "may pick a different convolution algorithm in every run -- turn it off")

    @contextlib.contextmanager
    def _determinism(self):
        """torch.use_deterministic_algorithms(True) for the duration of one call when the pipeline is deterministic."""
        if not self.deterministic:
            yield
            return
        self._check_deterministic_settings()
        prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
        torch.use_deterministic_algorithms(True)
        try:
            yield
        finally:
            torch.use_deterministic_algorithms(prev, warn_only=prev_warn)

    # ---- checkpoints, schedule ---------------------------------------------------------------------------------
    def save(self, prefix: str) -> None:
        torch.save(self.network.state_dict(), prefix + ".pt")
        torch.save(self.trainer.state_dict(), prefix + ".states.pt")

    def load(self, checkpoint: str) -> None:
        """A reference `.params` file (MXNet container, read without MXNet) or a state dict written by save()."""
        if checkpoint.endswith(".params"):
            mparams.load_checkpoint(self.network, checkpoint)
        else:
            self.network.load_state_dict(torch.load(checkpoint, map_location=self.device))

    def load_head(self, checkpoint: str) -> None:
        """Load a MaskFlownet-S checkpoint into the cascade's head (pipeline.py:59-60 -> MaskFlownet.load_head,
        network/MaskFlownet.py:409-410)."""
        head = getattr(self.network, "MaskFlownet_S", None)
        if head is None:
            raise MaskflowError("load_head: the network has no MaskFlownet_S head (only the cascade does)")
        if checkpoint.endswith(".params"):
            mparams.load_checkpoint(head, checkpoint)
        else:
            head.load_state_dict(torch.load(checkpoint, map_location=self.device))

    def fix_head(self) -> None:
        """Freeze the MaskFlownet-S head of the cascade (MaskFlownet.fix_head, network/MaskFlownet.py:412-414) and rebuild Adam
        over the cascade's own parameters.  Optional: without it train_batch trains the cascade end to end, head included."""
        head = getattr(self.network, "MaskFlownet_S", None)
        if head is None:
            raise MaskflowError("fix_head: the network has no MaskFlownet_S head (only the cascade does)")
        for p in head.parameters():
            p.requires_grad_(False)
        self._bucket = None
        self.trainer = torch.optim.Adam([p for p in self.network.parameters() if p.requires_grad], lr=self._lr)

    def set_learning_rate(self, steps: int) -> bool:
        i = 0
        while i < len(self.lr_schedule) and steps > self.lr_schedule[i][0]:
            i += 1
        try:
            lr = self.lr_schedule[i][1]
        except IndexError:
            return False
        for g in self.trainer.param_groups:
            g["lr"] = lr
        self._lr = lr
        return True

    @property
    def lr(self):
        return self._lr

    # ---- training ----------------------------------------------------------------------------------------------
    def loss(self, pred, occ_masks, labels, masks):
        return losses.multiscale_epe(labels, masks, pred, scales=self.strides, weights=self.multiscale_weights, eps=1e-8, q=self.q)

    def centralize(self, img1, img2):
        return network.centralize(img1, img2)

    def train_batch(self, img1, img2, label, geo_aug, color_aug, mask=None, global_batch: Optional[int] = None) -> Dict[str, float]:
        """One optimisation step on this rank's shard.  img1 / img2 (n,3,H,W) uint8, label (n,2,H,W) flow in (x,y) pixel
        order (flipped to the network's (y,x) after the augmentation, pipeline.py:106), mask (n,1,H,W) uint8 or None.
        global_batch: the batch size over ALL ranks (default: n * world size) -- what Trainer.step(batch_size) divides by.
        Returns {"epe": mean EPE of THIS rank's samples} (the reference averages over its context list in one process)."""
        with self._determinism():
            return self._train_batch(img1, img2, label, geo_aug, color_aug, mask, global_batch)

    def _train_batch(self, img1, img2, label, geo_aug, color_aug, mask, global_batch) -> Dict[str, float]:
        dev = self.device
        n = img1.shape[0]
        if mask is None:
            mask = np.full((n, 1, 1, 1), 255, dtype=np.uint8)
        img1, img2, mask = _to_device(img1, dev), _to_device(img2, dev), _to_device(mask, dev)
        label = _to_device(label, dev, torch.float32)
        self._begin_step()
        with torch.no_grad():                                   # the augmentation is data preparation (forward only)
            img1, img2, label, mask = geo_aug(img1, img2, label, mask)        # uint8 in: `/ 255` is folded into the kernel
            img1, img2 = color_aug(img1, img2)
            img1, img2, _ = self.centralize(img1, img2)
            label = label.flip(1).contiguous()
        pred, occ_masks, _ = self.network(img1, img2)
        per_sample = self.loss(pred, occ_masks, label, mask)
        self._finish_step(per_sample, n, global_batch)
        with torch.no_grad():
            epe = epe_loss_with_mask(ops.upsample(pred[-1].detach(), self.scale), label, mask)
        return {"epe": float(epe.mean().item())}

    def _begin_step(self) -> None:
        self.network.train()
        if self._bucket is None:
            self._bucket = mdist.GradBucket(self.network.parameters())
        self._bucket.zero_()

    def _finish_step(self, per_sample: torch.Tensor, n: int, global_batch: Optional[int]) -> None:
        """Backward of the summed per-sample losses, ONE gradient all-reduce scaled by 1/global_batch (default: n * world
        size), Adam step: the tail every training step shares."""
        per_sample.sum().backward()                             # per-sample losses are summed (pipeline.py:112-113)
        world = torch.distributed.get_world_size() if torch.distributed.is_initialized() else 1
        self._bucket.allreduce_(global_batch=n * world if global_batch is None else global_batch)
        self.trainer.step()                                     # trainer.step(batch_size): the 1/batch rescale is in the bucket

    def train_batch_unsupervised(self, img1, img2, color_aug=None, global_batch: Optional[int] = None) -> Dict[str, float]:
        """One unsupervised optimisation step on this rank's shard of unlabelled pairs (losses.unsupervised_loss: census
        photometric loss masked by the forward-backward check, plus smooth_weight times the second-order smoothness).
        img1 / img2 (n,3,H,W) uint8, H and W multiples of 64.  The network runs once at batch 2n on [img1; img2] ->
        [img2; img1]; color_aug (an augment.ColorAugmentation for batch n) changes only the network input, the losses see
        the original images.  global_batch: pairs over ALL ranks (default n * world size); each pair contributes both
        directions' losses.  Returns the means over this rank's 2n directed pairs: {"loss", "photo", "smooth",
        "occluded"} (occluded: share of pixels left out of the census term)."""
        with self._determinism():
            return self._train_batch_unsupervised(img1, img2, color_aug, global_batch)

    def _train_batch_unsupervised(self, img1, img2, color_aug, global_batch) -> Dict[str, float]:
        img1, img2 = _to_device(img1, self.device), _to_device(img2, self.device)
        if img1.dtype != torch.uint8 or img2.dtype != torch.uint8 or img1.dim() != 4 or img1.shape[1] != 3 \
                or img1.shape != img2.shape:
            raise MaskflowError(f"train_batch_unsupervised: expected two uint8 (n,3,H,W) batches of one shape, got "
                                f"{tuple(img1.shape)} {img1.dtype} and {tuple(img2.shape)} {img2.dtype}")
        n, _, H, W = img1.shape
        if H % 64 or W % 64:
            raise MaskflowError(f"train_batch_unsupervised: H and W must be multiples of 64, got {H}x{W}")
        self._begin_step()
        with torch.no_grad():
            a, b = img1.float() / 255.0, img2.float() / 255.0
            x1, x2 = (a, b) if color_aug is None else color_aug(a, b)
            x1, x2, _ = self.centralize(torch.cat([x1, x2]), torch.cat([x2, x1]))
        pred, _, _ = self.network(x1, x2)
        flow = ops.upsample(pred[-1], self.scale)
        out = losses.unsupervised_loss(a, b, flow[:n], flow[n:], self.smooth_weight)
        self._finish_step(out.loss, n, global_batch)
        means = torch.stack([t.detach().mean() for t in out]).tolist()
        return dict(zip(("loss", "occluded", "photo", "smooth"), means))

    # ---- inference ---------------------------------------------------------------------------------------------
    @torch.no_grad()
    def do_batch_mx(self, img1, img2, resize=None):
        """img1 / img2 in [0,1] float32 (or uint8): centralize, resize to multiples of 64 (or `resize`), network."""
        H, W = img1.shape[2:]
        if getattr(self.network, "inference_precision", "fp32") != self.precision:
            self.network.inference_precision = self.precision
        with self._determinism():
            a, b, _ = ops.preprocess(img1.contiguous(), img2.contiguous(), ops.padded_size(H, W, resize))
            return self.network(a, b)

    @torch.no_grad()
    def do_batch(self, img1, img2, label=None, mask=None, resize=None):
        with self._determinism():
            return self._do_batch(img1, img2, label, mask, resize)

    def _do_batch(self, img1, img2, label, mask, resize):
        H, W = img1.shape[2:]
        self.network.eval()
        flows, occ_masks, _ = self.do_batch_mx(img1, img2, resize=resize)
        flow = ops.postprocess(flows[-1], H, W, flip_channels=False, is_flow=True).permute(0, 3, 1, 2).contiguous()
        occ_mask = None
        if occ_masks and occ_masks[0] is not None and occ_masks[0].shape[1] == 1:
            occ_mask = ops.postprocess(occ_masks[0], H, W, flip_channels=False, is_flow=False).permute(0, 3, 1, 2).contiguous()
        img2f = img2.float() / 255.0 if img2.dtype == torch.uint8 else img2
        grid = ops.grid_generator_warp(flow.flip(1).contiguous()).clamp_(-1, 1)           # Reconstruction2DSmooth (layer.py:20-30)
        warp = ops.bilinear_sampler(img2f.contiguous(), grid)
        epe = None
        if label is not None and mask is not None:
            epe = epe_loss_with_mask(flow, label, mask)
        return flow, occ_mask, warp, epe

    @staticmethod
    def _stack(samples: Iterable[np.ndarray]) -> np.ndarray:
        return np.transpose(np.stack(list(samples), axis=0), (0, 3, 1, 2))

    @torch.no_grad()
    def validate(self, img1: List[np.ndarray], img2, label, mask=None, batch_size: int = 1, resize=None, return_type: str = "epe"):
        """Whole-dataset validation: lists of HWC arrays (uint8 images, float flow in (x,y), uint8 masks) -> mean EPE, or,
        for return_type != 'epe', the KITTI outlier ratio (error > 3 px and > 5 % of the label's magnitude)."""
        size, dev, out = len(img1), self.device, []
        if mask is None:
            mask = [np.full((1, 1, 1), 255, dtype=np.uint8)] * size
        for j in range(0, size, batch_size):
            a, b = _to_device(self._stack(img1[j:j + batch_size]), dev), _to_device(self._stack(img2[j:j + batch_size]), dev)
            labels = _to_device(self._stack(label[j:j + batch_size]), dev, torch.float32).flip(1).contiguous()
            masks = _to_device(self._stack(mask[j:j + batch_size]), dev, torch.float32) / 255.0
            masks = masks.expand(labels.shape[0], 1, labels.shape[2], labels.shape[3]).contiguous()
            flows, _, _, epe = self.do_batch(a, b, labels, masks, resize=resize)
            if return_type != "epe":
                err = (flows - labels).square().sum(dim=1, keepdim=True).sqrt()
                mag = labels.square().sum(dim=1, keepdim=True).sqrt()
                bad = ((err > 3) & ((err / (mag + 1e-8)) > 0.05)).float() * masks
                epe = bad.flatten(1).sum(dim=1) / masks.flatten(1).sum(dim=1)
            out.append(epe.cpu().numpy())
        return float(np.mean(np.concatenate(out, axis=0), axis=0))

    @torch.no_grad()
    def predict(self, img1: List[np.ndarray], img2, batch_size: int, resize=None):
        """Whole-dataset prediction: yields (flow (H,W,2) in (x,y) pixels, occlusion mask (H,W,1), warped second image
        (H,W,3)) per sample, as the reference's generator does."""
        size, dev = len(img1), self.device
        for j in range(0, size, batch_size):
            a, b = _to_device(self._stack(img1[j:j + batch_size]), dev), _to_device(self._stack(img2[j:j + batch_size]), dev)
            flow, occ_mask, warped, _ = self.do_batch(a, b, resize=resize)
            flow = flow.permute(0, 2, 3, 1).flip(-1).cpu().numpy()
            occ_mask = occ_mask.permute(0, 2, 3, 1).cpu().numpy() if occ_mask is not None else [None] * len(flow)
            warped = warped.permute(0, 2, 3, 1).cpu().numpy()
            for k in range(len(flow)):
                yield flow[k], occ_mask[k], warped[k]
