"""Host-side mirror of the reference's model graphs, calling the fused CUDA operators.

`MaskFlownetS` computes what `MaskFlownet_S.hybrid_forward` computes (network/MaskFlownet.py:197-315) and
`MaskFlownet` what the cascade computes (:443-545), but is organised around the hot path instead of transcribing the
unrolled reference code: one loop over pyramid levels in which

    Upsample(2) flow/mask + offset build + DeformableConvolution + sigmoid-mask multiply + trade-off + LeakyReLU
        (MaskFlownet.py:228-233)                                   -> one launch of ops.warp_mask      (K3)
    Correlation + LeakyReLU (:234-235), written straight into its slot of the decoder's concat buffer (:236)
                                                                    -> one launch of ops.correlation    (K1)
    Upsample(4) + GridGenerator + BilinearSampler + sigmoid-0.5 + concat (:308-313)
                                                                    -> one launch of ops.image_warp_concat (K5)

The dense 3x3 / transposed convolutions (about 98 % of the FLOPs, SURVEY.md section 0.4; row N2) run on the wgmma
kernel of csrc/conv3x3_wgmma.cu: f32 in / out, bf16 hi+lo split operands, fp32 accumulation.  At inference (`_fast`) with
in-place concat buffers and fused heads; with gradients enabled (`train_tc_forward`, default) every 3x3 convolution still
runs its FORWARD on that kernel and its backward through aten.convolution_backward (ops.conv3x3_train), the transposed
convolutions and the concats through torch autograd.  Sub-module names equal the reference's gluon prefixes (conv1a ... deform5, conv5f,
dc_conv7 ...) so that shipped .params checkpoints map by name (maskflownet_b200.params).

All flows are (y, x)-ordered and in units of pixels/scale, as in the reference (pipeline.py:105, MaskFlownet.py:69).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as tF

from . import camera, ops

PYRAMID_CH = {1: 16, 2: 32, 3: 64, 4: 96, 5: 128, 6: 196}   # network/MaskFlownet.py:79-96
DECODER_CH = (128, 128, 96, 64, 32)                           # convL_0 .. convL_4 (:102-130)
STRIDES = {6: 64, 5: 32, 4: 16, 3: 8, 2: 4}                   # self.strides (:71)
SLOPE = 0.1
PRECISIONS = ("fp32", "bf16")                                 # _FlowNetBase.inference_precision


def _conv(cin, cout, k=3, s=1, p=1, d=1):
    return nn.Conv2d(cin, cout, k, s, p, d)


def _swap_halves(t: torch.Tensor, n: int) -> torch.Tensor:
    """[t[n:]; t[:n]] of a (2n, ...) batch, in a new contiguous tensor: the second images of the reversed pairs."""
    return torch.cat([t[n:], t[:n]], dim=0)


def msra_prelu_init_(module: nn.Module, slope: float = SLOPE, seed: Optional[int] = None) -> None:
    """MSRAPrelu(factor_type='avg', slope) for weights, zeros for biases -- the reference's initialiser
    (network/pipeline.py:26)."""
    gen = torch.Generator().manual_seed(seed) if seed is not None else None
    for name, p in module.named_parameters():
        if p.dim() < 2:
            with torch.no_grad():
                p.zero_()
            continue
        hw = 1
        for d in p.shape[2:]:
            hw *= d
        fan_in, fan_out = p.shape[1] * hw, p.shape[0] * hw
        std = math.sqrt(2.0 / ((1 + slope ** 2) * (fan_in + fan_out) / 2.0))
        with torch.no_grad():
            p.copy_((torch.randn(p.shape, generator=gen) * std).to(p.device))


class DeformParams(nn.Module):
    """Weights of one layer.DeformableConv2D block (network/layer.py:32-110): weight (F, C, 3, 3) and bias (F)."""

    def __init__(self, channels: int, use_bias: bool = True):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(channels, channels, 3, 3))
        self.bias = nn.Parameter(torch.zeros(channels)) if use_bias else None


class _Slab:
    """Inference form of a dense block's output: its concat buffer as a split activation (ops.SplitAct), and -- when the
    block's last convolution also produced them -- the linear heads' partial sums over everything but that convolution's
    own last_oc output channels, in the fp32 tensor `prefix` (see _FlowNetBase._dense_split)."""

    def __init__(self, act: "ops.SplitAct", prefix: Optional[torch.Tensor], last_oc: int):
        self.act, self.prefix, self.last_oc = act, prefix, last_oc

    @property
    def channels(self) -> int:
        return self.act.channels


class _FlowNetBase(nn.Module):
    fuse_heads = True   # inference: pred_flow / pred_mask over the block input ride on conv{L}_4's input pass
    use_resample_warp = True   # inference: K3 through linearity (ops.warp_mask(resample=True)) at every level
    use_tc_conv = True   # inference: decoder / context 3x3 convolutions on the fp32-accurate tensor-core kernel (row N2)
    # training (grad enabled): the 3x3 convolutions still run their FORWARD on the wgmma kernel (ops.conv3x3_train: bias +
    # LeakyReLU fused, the output doubles as the activation mask), the BACKWARD is aten.convolution_backward (cuDNN fp32).
    # False: cuDNN both ways.
    train_tc_forward = True

    @property
    def inference_precision(self) -> str:
        """Arithmetic of the inference forward's 3x3 convolutions: "fp32" (default: the fp32-accurate bf16 hi/lo split)
        or "bf16" (opt-in: one bf16 product per multiply-add, fp32 accumulation, and the dense blocks' and context
        network's activations stored as bf16 -- ops.conv3x3_slices(bf16=True), include/maskflow_b200.h MFN_CONV_BF16).
        Correlation, warps, sampling and pre/post-processing stay fp32-accurate; training (autograd recording) is not
        affected.  Setting it on the cascade also sets it on its MaskFlownet_S head."""
        return self.__dict__.get("_inference_precision", "fp32")

    @inference_precision.setter
    def inference_precision(self, value: str) -> None:
        if value not in PRECISIONS:
            raise ops.MaskflowError(f"inference_precision must be one of {PRECISIONS}, got {value!r}")
        for m in self.modules():
            if isinstance(m, _FlowNetBase):
                m.__dict__["_inference_precision"] = value

    def _bf16(self) -> bool:
        return self.inference_precision == "bf16"

    def _packed(self, name):
        """Packed split-bf16 weight image of conv `name`, rebuilt when the parameter changes."""
        cache = self.__dict__.setdefault("_pack_cache", {})
        w = getattr(self, name).weight
        key = (w.data_ptr(), w._version)
        hit = cache.get(name)
        if hit is None or hit[0] != key:
            cache[name] = (key, ops.conv3x3_pack(w))
        return cache[name][1]

    def _packed_fn(self, key, params, build):
        """Cached derived tensors (fused / re-arranged weight images), rebuilt when any source parameter changes."""
        cache = self.__dict__.setdefault("_pack_cache", {})
        ver = tuple((p.data_ptr(), p._version) for p in params if p is not None)
        hit = cache.get(key)
        if hit is None or hit[0] != ver:
            cache[key] = (ver, build())
        return cache[key][1]

    def _head_convs(self, lvl, with_mask):
        pf = getattr(self, f"pred_flow{lvl}")
        pm = getattr(self, f"pred_mask{lvl}") if with_mask and hasattr(self, f"pred_mask{lvl}") else None
        return [pf] + ([pm] if pm is not None else [])

    def _heads(self, lvl, x, with_mask):
        """pred_flow{lvl} (2 channels) and pred_mask{lvl} (1 channel) read the same block output
        (network/MaskFlownet.py:224, 226 ...): inference runs them as ONE 3-output convolution, no activation -- and, when
        the dense block left their partial sums (a _Slab with a prefix tensor), only over the block's last 32 channels."""
        convs = self._head_convs(lvl, with_mask)
        pm = convs[1] if len(convs) > 1 else None
        if not isinstance(x, _Slab):
            return (self._conv_act(f"pred_flow{lvl}", x, 1.0),
                    self._conv_act(f"pred_mask{lvl}", x, 1.0) if pm is not None else None)
        nh = 2 + (1 if pm is not None else 0)
        N, _, H, W = x.act.shape
        dev = x.act.buf.device
        if x.prefix is not None and x.prefix.shape[1] >= nh:   # partial sums present: finish over conv{L}_4's output
            oc = x.last_oc

            def build_tail():
                w = torch.cat([c.weight.detach()[:, :oc] for c in convs], dim=0).contiguous()
                b = torch.cat([c.bias.detach() for c in convs], dim=0).contiguous()
                return ops.conv3x3_pack(w), b
            packed, b = self._packed_fn(f"heads_tail{lvl}", [p for c in convs for p in (c.weight, c.bias)], build_tail)
            y = torch.empty((N, nh, H, W), device=dev, dtype=torch.float32)
            ops.conv3x3_split(x.act, 0, oc, packed, b, nh, 1.0, out=y, bf16=self._bf16())
            y += x.prefix[:, :nh]
        else:
            def build():
                w = torch.cat([c.weight.detach() for c in convs], dim=0).contiguous()
                b = torch.cat([c.bias.detach() for c in convs], dim=0).contiguous()
                return ops.conv3x3_pack(w), b
            packed, b = self._packed_fn(f"heads{lvl}", [p for c in convs for p in (c.weight, c.bias)], build)
            y = torch.empty((N, nh, H, W), device=dev, dtype=torch.float32)
            ops.conv3x3_split(x.act, 0, x.channels, packed, b, nh, 1.0, out=y, bf16=self._bf16())
        if pm is None:
            return y, None
        return y[:, :2].contiguous(), y[:, 2:3].contiguous()

    def _upfeat(self, lvl, x):
        """feat = LeakyReLU(upfeat{lvl}(x)): ConvTranspose2d(4, 2, 1) as a 3x3 convolution + depth-to-space on the
        tensor-core kernel (ops.conv_transpose4x4_pack)."""
        up = getattr(self, f"upfeat{lvl}")
        if not isinstance(x, _Slab):
            return tF.leaky_relu(up(x), SLOPE)
        packed = self._packed_fn(f"upfeat{lvl}", [up.weight], lambda: ops.conv_transpose4x4_pack(up.weight))
        N, _, H, W = x.act.shape
        F = up.out_channels
        out = torch.empty((N, F, 2 * H, 2 * W), device=x.act.buf.device, dtype=torch.float32)
        ops.conv3x3_split(x.act, 0, x.channels, packed, up.bias, 4 * F, SLOPE, out=out, depth_to_space=True,
                          bf16=self._bf16())
        return out

    def _plain(self, name, x):
        """3x3 convolution without activation (conv{L}f, dc_conv7)."""
        conv = getattr(self, name)
        if not self._fast(x):
            return self._conv_act(name, x, 1.0)
        return ops.conv3x3(x, self._packed(name), conv.bias, conv.out_channels, 1.0, conv.dilation[0], bf16=self._bf16())

    def _conv_act(self, name, x, slope):
        """Autograd path of one 3x3 convolution (+ LeakyReLU when slope != 1): torch.nn.functional (cuDNN both ways), or --
        train_tc_forward -- the tensor-core forward with the cuDNN backward."""
        conv = getattr(self, name)
        if (self.train_tc_forward and x.is_cuda and conv.kernel_size == (3, 3) and conv.padding == conv.dilation
                and conv.stride[0] == conv.stride[1] and conv.groups == 1):
            return ops.conv3x3_train(x, conv.weight, conv.bias, self._packed(name), slope, conv.dilation[0], conv.stride[0])
        y = conv(x)
        return y if slope == 1.0 else tF.leaky_relu(y, slope)

    def _fast(self, x):
        return self.use_tc_conv and x.is_cuda and not (torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()))

    def _pyramid(self, x, names):
        """Six levels of (3x3 stride-2, 3x3, 3x3) convolutions + LeakyReLU (network/MaskFlownet.py:200-202).  Inference:
        all eighteen run on the wgmma convolution kernel (bias + activation fused)."""
        feats = []
        fast = self._fast(x)
        for lvl in range(1, 7):
            for j, sfx in enumerate(names):
                name = f"conv{lvl}{sfx}"
                conv = getattr(self, name)
                if fast:
                    x = ops.conv3x3(x, self._packed(name), conv.bias, conv.out_channels, SLOPE, 1, 2 if j == 0 else 1,
                                    bf16=self._bf16())
                else:
                    x = self._conv_act(name, x, SLOPE)
            feats.append(x)
        return feats  # [c?1 .. c?6]

    @staticmethod
    def _joined(im1, im2):
        """[im1; im2] as one (2N, ...) batch: a view when im1 and im2 are the two adjacent halves of one buffer
        (ops.preprocess), else a copy."""
        n = im1.shape[0]
        if (im1.is_contiguous() and im2.is_contiguous() and im1.shape == im2.shape and im1.dtype == im2.dtype
                and im1.untyped_storage().data_ptr() == im2.untyped_storage().data_ptr()
                and im2.storage_offset() == im1.storage_offset() + im1.numel()):
            return im1.view(-1).as_strided((2 * im1.numel(),), (1,)).view((2 * n,) + tuple(im1.shape[1:]))
        return torch.cat([im1, im2], dim=0)

    def _pyramid_pair(self, im1, im2, names, bidirectional=False):
        """Both images through the shared pyramid; inference batches them into one pass (half the launches).  When im1 and
        im2 are the two adjacent halves of one buffer (ops.preprocess), that buffer is the batch: no copy.
        bidirectional (inference only): the pairs (im1 -> im2) then (im2 -> im1) from the same pass -- c1 is the whole
        2N batch [f(im1); f(im2)] and c2 its halves swapped, [f(im2); f(im1)], one copy per level from level 2 on (no
        consumer reads level 1 of c2, which is None)."""
        if self._fast(im1):
            n = im1.shape[0]
            f = self._pyramid(self._joined(im1, im2), names)
            if bidirectional:
                return f, [None] + [_swap_halves(t, n) for t in f[1:]]
            return [t[:n] for t in f], [t[n:] for t in f]
        return self._pyramid(im1, names), self._pyramid(im2, names)

    def _check_bidirectional(self, im1, im2):
        if not self._fast(im1):
            raise ops.MaskflowError("bidirectional=True is an inference feature: it needs CUDA inputs, use_tc_conv and no "
                                    "autograd recording (call it under torch.no_grad())")
        if im1.shape != im2.shape:
            raise ops.MaskflowError(f"bidirectional: im1 {tuple(im1.shape)} and im2 {tuple(im2.shape)} differ")

    def _dense(self, lvl, x):
        """x = concat(leaky(conv_i(x)), x) five times (network/MaskFlownet.py:219-223 ...).  Inference: see _dense_split."""
        if self._fast(x):
            return self._dense_split(lvl, x)
        for i in range(5):
            x = torch.cat([self._conv_act(f"conv{lvl}_{i}", x, SLOPE), x], dim=1)
        return x

    def _dense_split(self, lvl, base):
        """Inference dense block.  One concat buffer in the split format (ops.SplitAct) holds [conv{lvl}_4 | ... |
        conv{lvl}_0 | base]: the fp32 base (correlation, features, flow) is packed into it once, and every convolution reads
        its input channels in place (a pure tensor copy per chunk) and writes its output, already split, in front of them.
        Every slice starts at a multiple of 16 channels.  With fuse_heads the last convolution also carries the linear
        heads over ITS input (everything the heads read except that convolution's own 32 output channels): weights
        [W_heads[:, 32:] ; 0 (to an even count) ; W_4]; the heads' partial sums go to a separate fp32 tensor (split storage
        would round them) -- one pass over the ~550-channel input instead of two.  Returns the block output as a _Slab."""
        N, Cb, H, W = base.shape
        front = sum(DECODER_CH)
        bf16 = self._bf16()
        act = ops.SplitAct(N, front + Cb, H, W, base.device, bf16=bf16)
        act.pack(base, front)
        nh = (2 + (1 if hasattr(self, f"pred_mask{lvl}") else 0)) if self.fuse_heads else 0
        lp = nh + nh % 2   # the kernel writes split channels in pairs: an even prefix
        prefix = None
        off = front
        for i, oc in enumerate(DECODER_CH):
            assert off % 16 == 0 and (off - oc) % 16 == 0
            conv = getattr(self, f"conv{lvl}_{i}")
            if i == len(DECODER_CH) - 1 and nh:
                heads = self._head_convs(lvl, True)

                def build():
                    w = conv.weight.detach()
                    w = torch.cat([h.weight.detach()[:, oc:] for h in heads] + [w.new_zeros((lp - nh,) + w.shape[1:]), w],
                                  dim=0).contiguous()
                    b = torch.cat([torch.zeros(lp, device=w.device), conv.bias.detach()]).contiguous()
                    return ops.conv3x3_pack(w), b
                packed, b = self._packed_fn(f"conv{lvl}_4+heads", [conv.weight, conv.bias] + [h.weight for h in heads], build)
                prefix = torch.empty((N, lp, H, W), device=base.device, dtype=torch.float32)
                ops.conv3x3_split(act, off, act.channels - off, packed, b, lp + oc, SLOPE, out=prefix, out_split=act,
                                  out_c0=off - oc, linear_prefix=lp, bf16=bf16)
            else:
                ops.conv3x3_split(act, off, act.channels - off, self._packed(f"conv{lvl}_{i}"), conv.bias, oc, SLOPE,
                                  out_split=act, out_c0=off - oc, bf16=bf16)
            off -= oc
        return _Slab(act, prefix, DECODER_CH[-1] if nh else 0)

    def _context(self, x):
        if isinstance(x, _Slab):
            # inference: dc_conv1 reads the block's split buffer in place, dc_conv1..6 chain in the split format, dc_conv7
            # writes the fp32 flow
            act = x.act
            N, _, H, W = act.shape
            bf16 = self._bf16()
            for i in range(1, 8):
                conv = getattr(self, f"dc_conv{i}")
                if i == 7:
                    y = torch.empty((N, conv.out_channels, H, W), device=act.buf.device, dtype=torch.float32)
                    ops.conv3x3_split(act, 0, act.channels, self._packed("dc_conv7"), conv.bias, conv.out_channels, 1.0,
                                      conv.dilation[0], out=y, bf16=bf16)
                    return y
                nxt = ops.SplitAct(N, conv.out_channels, H, W, act.buf.device, bf16=bf16)
                ops.conv3x3_split(act, 0, act.channels, self._packed(f"dc_conv{i}"), conv.bias, conv.out_channels, SLOPE,
                                  conv.dilation[0], out_split=nxt, bf16=bf16)
                act = nxt
        for i in range(1, 7):
            x = self._conv_act(f"dc_conv{i}", x, SLOPE)
        return self._plain("dc_conv7", x)

    def _make_decoder(self, in_ch: Dict[int, int], with_mask: bool, upfeat_ch):
        for lvl in (6, 5, 4, 3, 2):
            c = in_ch[lvl]
            for i, oc in enumerate(DECODER_CH):
                setattr(self, f"conv{lvl}_{i}", _conv(c, oc))
                c += oc
            setattr(self, f"pred_flow{lvl}", _conv(c, 2))
            if with_mask and lvl > 2:
                setattr(self, f"pred_mask{lvl}", _conv(c, 1))
            if lvl > 2:
                setattr(self, f"upfeat{lvl - 1}", nn.ConvTranspose2d(c, upfeat_ch[6 - lvl], 4, 2, 1))
        c2 = in_ch[2] + sum(DECODER_CH)
        dil = (1, 2, 4, 8, 16, 1)
        chs = (128, 128, 128, 96, 64, 32)
        c = c2
        for i in range(6):
            setattr(self, f"dc_conv{i + 1}", _conv(c, chs[i], 3, 1, dil[i], dil[i]))
            c = chs[i]
        self.dc_conv7 = _conv(c, 2)


class MaskFlownetS(_FlowNetBase):
    """MaskFlownet-S (reference class MaskFlownet_S, network/MaskFlownet.py:66-315)."""

    def __init__(self, flow_multiplier: float = 1.0, deform_bias: bool = True, upfeat_ch=(16, 16, 16, 16),
                 border_mode: int = ops.BORDER_MXNET15):
        super().__init__()
        self.scale = 20.0 * flow_multiplier
        self.md = 4
        self.border_mode = border_mode
        self.upfeat_ch = tuple(upfeat_ch)
        self.event_hook = None  # optional callable(kind, level, 0|1): bench.py brackets kernels with CUDA events
        cin = 3
        for lvl in range(1, 7):
            co = PYRAMID_CH[lvl]
            setattr(self, f"conv{lvl}a", _conv(cin, co, 3, 2))
            setattr(self, f"conv{lvl}b", _conv(co, co))
            setattr(self, f"conv{lvl}c", _conv(co, co))
            cin = co
        D = (2 * self.md + 1) ** 2
        in_ch = {6: D}
        for i, lvl in enumerate((5, 4, 3, 2)):
            in_ch[lvl] = D + PYRAMID_CH[lvl] + self.upfeat_ch[i] + 2
        self._make_decoder(in_ch, with_mask=True, upfeat_ch=self.upfeat_ch)
        for i, lvl in enumerate((5, 4, 3, 2)):
            setattr(self, f"deform{lvl}", DeformParams(PYRAMID_CH[lvl], deform_bias))
            setattr(self, f"conv{lvl}f", _conv(self.upfeat_ch[i], PYRAMID_CH[lvl]))
        msra_prelu_init_(self)

    # one correlation + its consumers' concat buffer: [corr | extras...]
    def _corr_block(self, lvl, f1, f2, extras: List[torch.Tensor]):
        N, _, H, W = f1.shape
        D = (2 * self.md + 1) ** 2
        # same gate as every other layer (_fast): with grad enabled and ANY trainable parameter the autograd operators
        # run, so a frozen pyramid + trainable decoder still trains conv{lvl}_0..4 (ADVICE r1)
        if not self._fast(f1):
            corr = ops.correlation(f1, f2, pad_size=self.md, max_displacement=self.md, leaky_slope=SLOPE)
            return self._dense(lvl, torch.cat([corr] + extras, dim=1) if extras else corr)
        tot = D + sum(e.shape[1] for e in extras)
        buf = torch.empty((N, tot, H, W), device=f1.device, dtype=torch.float32)
        hook = self.event_hook
        if hook is not None:
            hook("corr", lvl, 0)
        ops.correlation(f1, f2, pad_size=self.md, max_displacement=self.md, leaky_slope=SLOPE, out=buf[:, :D])
        if hook is not None:
            hook("corr", lvl, 1)
        c = D
        for e in extras:
            buf[:, c:c + e.shape[1]].copy_(e)
            c += e.shape[1]
        return self._dense(lvl, buf)

    def forward(self, im1: torch.Tensor, im2: torch.Tensor, want_cascade_inputs: bool = False,
                bidirectional: bool = False):
        """Returns (predictions [flow6..flow2, each * scale], [sigmoid(mask2)], srcs or None) like the reference
        (network/MaskFlownet.py:302-315).  srcs (needed only by the cascade) is built when want_cascade_inputs.
        bidirectional (inference only): im1 and im2 hold N images each and the outputs hold 2N pairs, (im1 -> im2) then
        (im2 -> im1), from one pyramid pass over [im1; im2] (_pyramid_pair)."""
        if bidirectional:
            self._check_bidirectional(im1, im2)
            n = im1.shape[0]
            im1 = self._joined(im1, im2)
            im2 = _swap_halves(im1, n) if want_cascade_inputs else None
            c1, c2 = self._pyramid_pair(im1[:n], im1[n:], "abc", bidirectional=True)
        else:
            c1, c2 = self._pyramid_pair(im1, im2, "abc")
        x = self._corr_block(6, c1[5], c2[5], [])   # correlation + dense block
        flow, mask = self._heads(6, x, True)
        flows = [flow]
        for lvl in (5, 4, 3, 2):
            feat = self._upfeat(lvl, x)
            dp = getattr(self, f"deform{lvl}")
            trade = self._plain(f"conv{lvl}f", feat)
            if self.event_hook is not None:
                self.event_hook("warp", lvl, 0)
            warp, flow_up, _ = ops.warp_mask(c2[lvl - 1], flow, mask, dp.weight, dp.bias, trade, self.scale,
                                             float(STRIDES[lvl]), 2, SLOPE, self.border_mode,
                                             # inference: every level is evaluated exactly through linearity (extended 3x3
                                             # convolution on wgmma + bilinear re-sampling + border-band tables, warp_lin.cu)
                                             packed_weight=self._packed(f"deform{lvl}") if self._fast(flow) else None,
                                             resample=self.use_resample_warp)
            if self.event_hook is not None:
                self.event_hook("warp", lvl, 1)
            x = self._corr_block(lvl, c1[lvl - 1], warp, [c1[lvl - 1], feat, flow_up])
            dflow, m = self._heads(lvl, x, lvl > 2)
            flow = flow_up + dflow
            if lvl > 2:
                mask = m
            else:
                mask_up2 = _  # Upsample(2)(mask3): the level-2 occlusion mask (network/MaskFlownet.py:283)
            flows.append(flow)
        flows[-1] = flow = flow + self._context(x)
        preds = [f * self.scale for f in flows]
        occ = [torch.sigmoid(mask_up2)]
        srcs = None
        if want_cascade_inputs:
            c30, c40 = ops.image_warp_concat(im1, im2, flow, mask_up2, self.scale)
            # quirk kept from the reference: levels 2 and 3 of c2s carry IMAGE-1 features (MaskFlownet.py:306)
            c2s = [c2[0], c1[1], c1[2], c2[3], c2[4], c2[5]]
            srcs = (c1, c2s, flows, c30, c40)
        return preds, occ, srcs


class MaskFlownet(_FlowNetBase):
    """Full cascade (reference class MaskFlownet, network/MaskFlownet.py:318-545): the S head plus a second, dual
    pyramid on [im1; 0] and [warp(im2); mask] with md=2 correlations."""

    def __init__(self, flow_multiplier: float = 1.0, deform_bias: bool = True, upfeat_ch=(16, 16, 16, 16),
                 border_mode: int = ops.BORDER_MXNET15):
        super().__init__()
        self.scale = 20.0 * flow_multiplier
        self.md = 2
        self.border_mode = border_mode
        self.MaskFlownet_S = MaskFlownetS(flow_multiplier, deform_bias, upfeat_ch, border_mode)
        cin = 4
        for lvl in range(1, 7):
            co = PYRAMID_CH[lvl]
            setattr(self, f"conv{lvl}x", _conv(cin, co, 3, 2))
            setattr(self, f"conv{lvl}y", _conv(co, co))
            setattr(self, f"conv{lvl}z", _conv(co, co))
            cin = co
        D = (2 * self.md + 1) ** 2
        in_ch = {6: 2 * D + 2}
        for i, lvl in enumerate((5, 4, 3, 2)):
            in_ch[lvl] = PYRAMID_CH[lvl] + upfeat_ch[i] + 2 * D + 4
        self._make_decoder(in_ch, with_mask=False, upfeat_ch=tuple(upfeat_ch))
        for lvl in (6, 5, 4, 3, 2):
            setattr(self, f"deform{lvl}", DeformParams(PYRAMID_CH[lvl], deform_bias))
        msra_prelu_init_(self)

    def _corr(self, a, b):
        return ops.correlation(a, b, pad_size=self.md, max_displacement=self.md, leaky_slope=SLOPE)

    def forward(self, im1, im2, bidirectional: bool = False):
        """As MaskFlownetS.forward; bidirectional: 2N pairs, (im1 -> im2) then (im2 -> im1), the head's pyramid computed
        once, the dual pyramid and decoder at batch 2N."""
        if bidirectional:
            self._check_bidirectional(im1, im2)
        _, _, srcs = self.MaskFlownet_S(im1, im2, want_cascade_inputs=True, bidirectional=bidirectional)
        c1, c2, flows_s, c30, c40 = srcs
        c3 = self._pyramid(c30, "xyz")
        c4 = self._pyramid(c40, "xyz")
        flow = flows_s[0]
        dp = self.deform6
        fast = self._fast(flow)
        warp, _, _ = ops.warp_mask(c2[5], flow, None, dp.weight, dp.bias, None, self.scale, float(STRIDES[6]), 1,
                                   SLOPE, self.border_mode, packed_weight=self._packed("deform6") if fast else None,
                                   resample=self.use_resample_warp)
        x = self._dense(6, torch.cat([self._corr(c1[5], warp), self._corr(c3[5], c4[5]), flow], dim=1))
        flow = flow + self._heads(6, x, False)[0]
        flows = [flow]
        for i, lvl in enumerate((5, 4, 3, 2)):
            feat = self._upfeat(lvl, x)
            dp = getattr(self, f"deform{lvl}")
            warp, flow_up, _ = ops.warp_mask(c2[lvl - 1], flow, None, dp.weight, dp.bias, None, self.scale,
                                             float(STRIDES[lvl]), 2, SLOPE, self.border_mode,
                                             packed_weight=self._packed(f"deform{lvl}") if fast else None,
                                             resample=self.use_resample_warp)
            x = self._dense(lvl, torch.cat([c1[lvl - 1], feat, self._corr(c1[lvl - 1], warp),
                                            self._corr(c3[lvl - 1], c4[lvl - 1]), flow_up, flows_s[i + 1]], dim=1))
            flow = flow_up + self._heads(lvl, x, False)[0]
            flows.append(flow)
        flows[-1] = flow = flow + self._context(x)
        return [f * self.scale for f in flows], [flow[:, 0:1]], []


# ---------------------------------------------------------------------------------------------------------------
# the step either side of the network: what PipelineFlownet.do_batch does around it (network/pipeline.py:85-87,117-147)
# ---------------------------------------------------------------------------------------------------------------
def centralize(img1: torch.Tensor, img2: torch.Tensor):
    """Subtract the per-sample RGB mean over both images (network/pipeline.py:85-87)."""
    mean = torch.cat([img1, img2], dim=2).mean(dim=(2, 3), keepdim=True)
    return img1 - mean, img2 - mean, mean


@torch.no_grad()
def predict_flow(net: nn.Module, img1_u8: torch.Tensor, img2_u8: torch.Tensor) -> torch.Tensor:
    """uint8 image pairs (N,3,H,W), H and W multiples of 64 -> full-resolution flow (N,2,H,W), (y,x)-ordered, in pixels:
    /255, centralize, network, Upsample(4) of the finest prediction (network/pipeline.py:99,117-138)."""
    if img1_u8.is_cuda and img1_u8.dtype == torch.uint8 and img1_u8.is_contiguous() and img2_u8.is_contiguous():
        a, b, _ = ops.preprocess(img1_u8, img2_u8)        # /255 + centralize in one fused op (csrc/prepost.cu)
    else:
        a, b, _ = centralize(img1_u8.float() / 255.0, img2_u8.float() / 255.0)
    preds = net(a, b)[0]
    return ops.upsample(preds[-1], 4)


@torch.no_grad()
def predict(net: nn.Module, img1: torch.Tensor, img2: torch.Tensor, resize=None):
    """PipelineFlownet.predict for one batch (network/pipeline.py:189-223), fused: uint8 (or [0,1] float) pairs (N,3,H,W) of
    ANY size -> /255 + centralize + BilinearResize2D to multiples of 64 (one op) -> network -> Upsample(4) + resize back +
    per-channel rescale + NHWC + (y,x)->(x,y) flip (one op).  Returns (flow (N,H,W,2) in (x,y) pixels -- the .flo layout,
    occlusion mask (N,H,W,1))."""
    N, _, H, W = img1.shape
    a, b, _ = ops.preprocess(img1, img2, ops.padded_size(H, W, resize))
    preds, occ, _ = net(a, b)
    flow = ops.postprocess(preds[-1], H, W, flip_channels=True, is_flow=True)
    mask = ops.postprocess(occ[0], H, W, flip_channels=False, is_flow=False) if occ and occ[0].shape[1] == 1 and \
        occ[0].shape[2] * 4 == a.shape[2] else None
    return flow, mask


def _pair_flows(net: nn.Module, img1: torch.Tensor, img2: torch.Tensor, resize, bidirectional: bool) -> torch.Tensor:
    """preprocess -> forward -> postprocess of the finest flow: (N,H,W,2) (x,y) flows of pairs (N,3,H,W), or with
    bidirectional (2N,H,W,2), img1 -> img2 then img2 -> img1."""
    _, _, H, W = img1.shape
    a, b, _ = ops.preprocess(img1, img2, ops.padded_size(H, W, resize))
    preds = net(a, b, bidirectional=True)[0] if bidirectional else net(a, b)[0]
    return ops.postprocess(preds[-1], H, W, flip_channels=True, is_flow=True)


def _frame_pair_flows(net: nn.Module, F: torch.Tensor, resize, bidirectional: bool) -> torch.Tensor:
    """_pair_flows of the B pairs (F[j], F[j+1]) of a frame buffer F (B+1,H,W,3) uint8: B flows, or 2B."""
    B = F.shape[0] - 1
    x = F.permute(0, 3, 1, 2).contiguous()
    return _pair_flows(net, x[:B], x[1:], resize, bidirectional)


@torch.no_grad()
def predict_bidirectional(net: nn.Module, img1: torch.Tensor, img2: torch.Tensor, resize=None, alpha: float = 0.01,
                          beta: float = 0.5):
    """Flow in both directions and forward-backward occlusion masks of uint8 (or [0,1] float) pairs (N,3,H,W) of any size.

    The mask `predict` returns is not a visibility map: for the cascade it is the y-component of the flow (the reference's
    "visual" output), for MaskFlownet-S the sigmoid of the learned warp mask.  This function gives one: a pixel is
    occluded (1) where its flow has no consistent match in the other direction's flow (ops.flow_consistency, Sundaram
    et al. 2010, constants alpha and beta).

    One ops.preprocess, one bidirectional forward (the pair's feature pyramid computed once for both directions), one
    ops.postprocess over the 2N finest flows, one ops.flow_consistency.  Returns (flow_fw, flow_bw, occ_fw, occ_bw) at the
    input size: flows (N,H,W,2) in (x,y) pixels, img1 -> img2 and img2 -> img1; masks (N,H,W) uint8, of img1's and of
    img2's pixels."""
    N = img1.shape[0]
    flows = _pair_flows(net, img1, img2, resize, True)
    flow_fw, flow_bw = flows[:N], flows[N:]
    occ_fw, occ_bw = ops.flow_consistency(flow_fw, flow_bw, alpha, beta)
    return flow_fw, flow_bw, occ_fw, occ_bw


@torch.no_grad()
def interpolate_frames(net: nn.Module, img1: torch.Tensor, img2: torch.Tensor, times, resize=None, alpha: float = 0.01,
                       beta: float = 0.5, occ_weight: float = 0.01) -> torch.Tensor:
    """In-between frames of uint8 pairs (N,3,H,W) of any size at the given times in (0,1) (0 = img1): predict_bidirectional
    (flows both ways and the occlusion masks, constants alpha, beta), then ops.interpolate_frames (occlusion-weighted
    forward splatting, occluded pixels weighted by occ_weight) on NHWC views of the images.  Returns (N,T,H,W,3) uint8, in
    the channel order of the inputs."""
    if img1.dtype != torch.uint8 or img2.dtype != torch.uint8:
        raise ops.MaskflowError(f"interpolate_frames: the images must be uint8, got {img1.dtype} and {img2.dtype}")
    ts = ops._interp_times(times, "interpolate_frames")
    flow_fw, flow_bw, occ_fw, occ_bw = predict_bidirectional(net, img1, img2, resize, alpha, beta)
    a = img1.permute(0, 2, 3, 1).contiguous()
    b = img2.permute(0, 2, 3, 1).contiguous()
    return ops.interpolate_frames(a, b, flow_fw, flow_bw, occ_fw, occ_bw, ts, occ_weight)


def _check_clip(clip, batch: int, who: str, name: str = "clip") -> None:
    if not isinstance(clip, torch.Tensor) or clip.dtype != torch.uint8 or clip.dim() != 4 or clip.shape[3] != 3:
        raise ops.MaskflowError(f"{who}: {name} must be a (T,H,W,3) uint8 tensor")
    if batch < 1:
        raise ops.MaskflowError(f"{who}: batch must be >= 1, got {batch}")


def _clip_batches(clip: torch.Tensor, batch: int):
    """(k0, nb, F) per batch of a clip's pairs: F holds frames k0 .. k0 + batch, padded with the last frame as the
    streamed classes pad it, and nb of its pairs are real."""
    P = clip.shape[0] - 1
    for k0 in range(0, P, batch):
        yield k0, min(batch, P - k0), clip[[min(k0 + j, P) for j in range(batch + 1)]]


def _track_batch(st, F: torch.Tensor, flows: torch.Tensor, n: int, xy=None, status=None, dropped=None):
    """ops.track_texture of F (B+1,H,W,3), then for pairs j < n track_advance along its 2B flows and track_seed of frame
    j + 1 into row j of xy, status and dropped (B rows allocated when not given)."""
    B = F.shape[0] - 1
    lam, lmax = ops.track_texture(F, st.spacing)
    if xy is None:
        xy = torch.empty((B, st.K, 2), dtype=torch.float32, device=F.device)
        status = torch.empty((B, st.K), dtype=torch.uint8, device=F.device)
        dropped = torch.empty((B,), dtype=torch.int32, device=F.device)
    for j in range(n):
        ops.track_advance(st, flows[j], flows[B + j])
        ops.track_seed(st, lam[j + 1], lmax[j + 1:j + 2], xy[j], status[j], dropped[j:j + 1])
    return xy, status, dropped


def _segment_batch(flows: torch.Tensor, carry, alpha: float, beta: float, kw: dict):
    """segment_motion's rule for a batch's first B frames from its 2B flows.  carry: the previous batch's last backward
    residual and mask (frame 0's side b), overwritten with this batch's.  Returns (segment_motion's four results, the
    backward residuals, the backward masks)."""
    B = flows.shape[0] // 2
    occ_fw, occ_bw = ops.flow_consistency(flows[:B], flows[B:], alpha, beta)
    affine, _, res = ops.affine_motion(flows, want_residual=True)
    res_b = torch.cat([carry[0], res[B:2 * B - 1]])
    occ_b = torch.cat([carry[1], occ_bw[:B - 1]])
    out = ops.segment_motion(res[:B], occ_fw, res_b, occ_b, flows[:B], affine[:B], **kw)
    carry[0].copy_(res[2 * B - 1:])
    carry[1].copy_(occ_bw[B - 1:])
    return out, res[B:], occ_bw


def _segment_last(res_bw, occ_bw, nb: int, shape, kw: dict):
    """The last frame from side b alone, row nb - 1 of the last batch's; with no pair (res_bw None) an empty frame."""
    if res_bw is None:
        return ops.segment_motion(shape=shape, **kw)
    return ops.segment_motion(res_b=res_bw[nb - 1:nb], occ_b=occ_bw[nb - 1:nb], **kw)


@torch.no_grad()
def track_video(net: nn.Module, frames: torch.Tensor, batch: int = 8, resize=None, spacing: int = 8, tau: float = 0.001,
                alpha: float = 0.01, beta: float = 0.5, boundary=(0.01, 0.002), max_tracks=None, queries=None):
    """Dense point tracks through a clip of uint8 frames (T,H,W,3) on the device, any channel order (ops.TrackState
    for the arguments; include/maskflow_b200.h, "Dense point tracking").  Frame 0 is seeded; then the pairs go through
    the bidirectional forward `batch` at a time (the last batch padded with the last frame, as video.VideoTracker does),
    the texture of each batch's frames in one ops.track_texture, and per pair ops.track_advance and ops.track_seed.  This
    is the eager chain VideoTracker captures.  Returns (xy (T,K,2) float32, status (T,K) uint8, dropped (T,) int32) on the
    device: every slot's position and status in every frame, and the seeding candidates left without a slot."""
    _check_clip(frames, batch, "track_video", "frames")
    T, H, W, _ = frames.shape
    st = ops.TrackState(H, W, spacing, tau, alpha, beta, boundary, max_tracks, queries, device=frames.device)
    xy = torch.empty((T, st.K, 2), dtype=torch.float32, device=frames.device)
    status = torch.empty((T, st.K), dtype=torch.uint8, device=frames.device)
    dropped = torch.empty((T,), dtype=torch.int32, device=frames.device)
    ops.track_start(st, frames[0].contiguous(), xy[0], status[0], dropped[0:1])
    for k0, nb, F in _clip_batches(frames, batch):
        flows = _frame_pair_flows(net, F, resize, True)
        _track_batch(st, F, flows, nb, xy[k0 + 1:], status[k0 + 1:], dropped[k0 + 1:])
    return xy, status, dropped


@torch.no_grad()
def stabilize_video(net: nn.Module, clip: torch.Tensor, batch: int = 8, resize=None, radius: int = 15, crop: float = 0.9,
                    iterations: int = ops.AFFINE_ITERATIONS, sigma: float = ops.AFFINE_SIGMA):
    """A stabilised clip of uint8 frames (T,H,W,3) on the device, any channel order.  The pairs go through the network
    `batch` at a time (the last batch padded with the last frame, as video.VideoStabilizer does) and each batch's flows
    through ops.affine_motion(iterations, sigma); camera.camera_path smooths the camera path over `radius` frames and
    zooms by `crop` (camera.stabilize_path states the rule; a pair whose fit failed, ok False, counts as no motion); one
    ops.warp_frames_affine warps every frame.  This is the eager chain VideoStabilizer streams.  Returns (stabilised clip
    (T,H,W,3) uint8 on the device, affine (T-1,2,3) float64 and ok (T-1,) bool on the device, M (T,2,3) float64 on the
    host: the warp of each frame, output pixel -> source position)."""
    _check_clip(clip, batch, "stabilize_video")
    camera.check_path_args(radius, crop, "stabilize_video")
    T, H, W, _ = clip.shape
    dev = clip.device
    P = T - 1
    affine = torch.empty((max(P, 0), 2, 3), dtype=torch.float64, device=dev)
    ok = torch.empty((max(P, 0),), dtype=torch.bool, device=dev)
    for k0, nb, F in _clip_batches(clip, batch):
        a, g = ops.affine_motion(_frame_pair_flows(net, F, resize, False), iterations, sigma)
        affine[k0:k0 + nb], ok[k0:k0 + nb] = a[:nb], g[:nb]
    M = camera.camera_path(affine.cpu().numpy(), ok.cpu().numpy(), H, W, radius, crop)
    out = ops.warp_frames_affine(clip.contiguous(), torch.from_numpy(M).to(dev))
    return out, affine, ok, M


@torch.no_grad()
def segment_motion(net: nn.Module, clip: torch.Tensor, batch: int = 8, resize=None, tau_lo: float = ops.SEG_TAU_LO,
                   tau_hi: float = ops.SEG_TAU_HI, min_area: int = ops.SEG_MIN_AREA,
                   max_objects: int = ops.SEG_MAX_OBJECTS, alpha: float = 0.01, beta: float = 0.5):
    """The objects moving relative to the camera in every frame of a clip of uint8 frames (T,H,W,3) on the device, any
    channel order (ops.segment_motion states the rule).  The pairs go through the bidirectional forward `batch` at a time
    (the last batch padded with the last frame, as video.VideoMotionSegmenter does); each batch's 2B flows through one
    ops.affine_motion(want_residual=True) at its defaults, and one ops.segment_motion segments the batch's first frames:
    frame k0 + j takes side a from pair j and side b from pair j - 1, or for j = 0 from the previous batch's last pair
    (for frame 0: none, given as NaN residuals, which are undefined).  The last frame is segmented from side b alone.  A
    one-frame clip gives one empty frame.  This is the eager chain VideoMotionSegmenter captures.
    Returns (labels (T,H,W) uint8, objects (T,max_objects,10) float64, count (T,) int32, dropped (T,) int32) on the
    device."""
    _check_clip(clip, batch, "segment_motion")
    ops.check_segment_args(tau_lo, tau_hi, min_area, max_objects, "segment_motion")
    T, H, W, _ = clip.shape
    dev = clip.device
    kw = dict(tau_lo=tau_lo, tau_hi=tau_hi, min_area=min_area, max_objects=max_objects)
    results = (torch.empty((T, H, W), dtype=torch.uint8, device=dev),
               torch.empty((T, max_objects, 10), dtype=torch.float64, device=dev),
               torch.empty((T,), dtype=torch.int32, device=dev), torch.empty((T,), dtype=torch.int32, device=dev))
    P = T - 1
    if P == 0:
        with torch.cuda.device(dev):
            last = _segment_last(None, None, 0, (1, H, W), kw)
    elif P > 0:
        carry = (torch.full((1, H, W), float("nan"), dtype=torch.float32, device=dev),
                 torch.zeros((1, H, W), dtype=torch.uint8, device=dev))
        for k0, nb, F in _clip_batches(clip, batch):
            out, res_bw, occ_bw = _segment_batch(_frame_pair_flows(net, F, resize, True), carry, alpha, beta, kw)
            for dst, src in zip(results, out):
                dst[k0:k0 + nb] = src[:nb]
        last = _segment_last(res_bw, occ_bw, nb, None, kw)      # side b of the last real pair
    else:                                                       # an empty clip
        return results
    for dst, src in zip(results, last):
        dst[P:] = src
    return results


@torch.no_grad()
def denoise_video(net: nn.Module, clip: torch.Tensor, batch: int = 8, resize=None, radius: int = ops.DENOISE_RADIUS,
                  sigma=None, h: float = ops.DENOISE_H, patch: int = ops.DENOISE_PATCH, alpha: float = 0.01,
                  beta: float = 0.5):
    """A denoised clip of uint8 frames (T,H,W,3) on the device, any channel order (ops.denoise_frames states the rule).
    The pairs go through the bidirectional forward `batch` at a time (the last batch padded with the last frame, as
    video.VideoDenoiser does), then one ops.denoise_frames over the whole clip averages each frame with up to `radius`
    neighbours on each side along the chained flow.  sigma=None takes ops.median_noise of the clip's first
    min(T, batch + 1) frames, the frames the stream sees first.  A one-frame clip comes back unchanged.  This is the
    eager chain VideoDenoiser streams.  Returns (denoised clip (T,H,W,3) uint8 on the device, the sigma used)."""
    _check_clip(clip, batch, "denoise_video")
    ops.check_denoise_args(radius, sigma, h, patch, alpha, beta, "denoise_video", sigma_optional=True)
    T, H, W, _ = clip.shape
    clip = clip.contiguous()
    if sigma is None:
        sigma = ops.median_noise(clip[:min(T, batch + 1)])
    if T == 1:
        return clip.clone(), float(sigma)
    fw = torch.zeros((T, H, W, 2), dtype=torch.float32, device=clip.device)   # slot T-1 (no pair) is never read
    bw = torch.zeros_like(fw)
    for k0, nb, F in _clip_batches(clip, batch):
        flows = _frame_pair_flows(net, F, resize, True)
        fw[k0:k0 + nb], bw[k0:k0 + nb] = flows[:nb], flows[batch:batch + nb]
    out = ops.denoise_frames(clip, fw, bw, radius, sigma, h, patch, alpha, beta)
    return out, float(sigma)


def precision_key(net: nn.Module) -> Tuple[str, ...]:
    """The inference_precision of every flow network inside `net` (the cascade's head may be set on its own): what a
    captured graph depends on besides the input shape."""
    return tuple(m.inference_precision for m in net.modules() if isinstance(m, _FlowNetBase))


class FlowPredictor:
    """predict_flow captured in a CUDA graph: one graph per input shape (and precision_key of the model), static uint8
    input buffers, one cudaGraphLaunch per call (the eager step is ~115 dependent launches; the graph removes the launch
    gaps between them).  After a precision switch the next call captures (or reuses) a graph of the new precision.
    Weights are read through the packed images cached in the model: call invalidate() after changing parameters.
    The returned tensor is the graph's STATIC output buffer: the next call overwrites it -- clone() it (or copy it to the
    host) before calling again if the previous result is still needed."""

    def __init__(self, net: nn.Module, warmup: int = 2):
        self.net, self.warmup, self._graphs = net, warmup, {}

    def invalidate(self) -> None:
        self._graphs.clear()

    @torch.no_grad()
    def __call__(self, img1_u8: torch.Tensor, img2_u8: torch.Tensor) -> torch.Tensor:
        dev = next(self.net.parameters()).device      # inputs may live on the host (pinned): the static buffers do not
        key = (tuple(img1_u8.shape), img1_u8.dtype, precision_key(self.net))
        entry = self._graphs.get(key)
        if entry is None:
            in1 = torch.empty(img1_u8.shape, dtype=img1_u8.dtype, device=dev)
            in2 = torch.empty(img2_u8.shape, dtype=img2_u8.dtype, device=dev)
            in1.copy_(img1_u8)
            in2.copy_(img2_u8)
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):      # warm-up off the capture: weight packing, kernel attributes, cuDNN-free path
                for _ in range(self.warmup):
                    predict_flow(self.net, in1, in2)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = predict_flow(self.net, in1, in2)
            entry = self._graphs[key] = (graph, in1, in2, out)
        graph, in1, in2, out = entry
        in1.copy_(img1_u8, non_blocking=True)
        in2.copy_(img2_u8, non_blocking=True)
        graph.replay()
        return out



class PipelinedFlowPredictor:
    """Serving loop around FlowPredictor for HOST buffers: every call enqueues (asynchronously)
        pinned uint8 images --H2D (copy stream)--> staging --D2D--> graph inputs --graph replay--> flow --D2D--> staging
        --D2H (copy stream)--> pinned fp32 flow
    with `depth` staging slots, so the H2D copy of request i+1 and the D2H copy of result i-1 run under the forward of
    request i (PCIe is full duplex; 22 MB in / 29 MB out per batch of 8 at 1024x448).
    One set of slots per input shape (and dtype), keyed like FlowPredictor's graphs: requests of different batch sizes or
    frame sizes may be interleaved, and each shape's slots rotate on their own.
    Results are complete after synchronize() (or after waiting on the event infer() returns)."""

    def __init__(self, net: nn.Module, depth: int = 2):
        self.pred = FlowPredictor(net)
        self.depth = depth
        self._slots = {}          # (shape, dtype) -> [slots of that shape, requests enqueued with it]
        self.h2d = self.d2h = None

    def _setup(self, img1, dev):
        shp = tuple(img1.shape)
        N, _, H, W = shp
        if self.h2d is None:
            self.h2d, self.d2h = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
        slots = []
        for _ in range(self.depth):
            slots.append({
                "in1": torch.empty(shp, dtype=img1.dtype, device=dev), "in2": torch.empty(shp, dtype=img1.dtype, device=dev),
                "out": torch.empty((N, 2, H, W), dtype=torch.float32, device=dev),
                "ev_h2d": torch.cuda.Event(), "ev_in_free": torch.cuda.Event(), "ev_out": torch.cuda.Event(),
                "ev_out_free": torch.cuda.Event(), "used": False})
        # the slots come from the allocator on the current stream (their memory may still be in use there, and under
        # torch.use_deterministic_algorithms a fill is queued on it): the copy streams start after that
        cur = torch.cuda.current_stream(dev)
        self.h2d.wait_stream(cur)
        self.d2h.wait_stream(cur)
        return [slots, 0]

    @torch.no_grad()
    def infer(self, img1_host: torch.Tensor, img2_host: torch.Tensor, out_host: torch.Tensor) -> torch.cuda.Event:
        dev = next(self.pred.net.parameters()).device
        if img2_host.shape != img1_host.shape or img2_host.dtype != img1_host.dtype:
            raise ValueError(f"infer: img1 {tuple(img1_host.shape)} and img2 {tuple(img2_host.shape)} differ")
        key = (tuple(img1_host.shape), img1_host.dtype)
        entry = self._slots.get(key)
        if entry is None:
            entry = self._slots[key] = self._setup(img1_host, dev)
        N, _, H, W = key[0]
        if tuple(out_host.shape) != (N, 2, H, W):
            raise ValueError(f"infer: out_host is {tuple(out_host.shape)}, the flow of this request is {(N, 2, H, W)}")
        s = entry[0][entry[1] % self.depth]
        entry[1] += 1
        cur = torch.cuda.current_stream(dev)
        with torch.cuda.stream(self.h2d):
            if s["used"]:
                self.h2d.wait_event(s["ev_in_free"])
            s["in1"].copy_(img1_host, non_blocking=True)
            s["in2"].copy_(img2_host, non_blocking=True)
            s["ev_h2d"].record(self.h2d)
        cur.wait_event(s["ev_h2d"])
        flow = self.pred(s["in1"], s["in2"])          # D2D into the graph's static inputs + replay
        s["ev_in_free"].record(cur)
        if s["used"]:
            cur.wait_event(s["ev_out_free"])
        s["out"].copy_(flow, non_blocking=True)
        s["ev_out"].record(cur)
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(s["ev_out"])
            out_host.copy_(s["out"], non_blocking=True)
            s["ev_out_free"].record(self.d2h)
        s["used"] = True
        return s["ev_out_free"]

    def synchronize(self) -> None:
        if self.h2d is not None:
            self.h2d.synchronize()
            self.d2h.synchronize()
        torch.cuda.current_stream().synchronize()
