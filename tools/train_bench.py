"""Training-step benchmark for BASELINE configs[2] (MaskFlownet-S forward+backward, batch 8, 512x384, 1 GPU) and configs[4]
(batch 32 sharded over the ranks, one NCCL gradient all-reduce per step; 960x540 pads to 960x576 like do_batch_mx).

    python tools/train_bench.py --hw 384x512 --batch 8 --steps 5
    torchrun --nproc-per-node 2 tools/train_bench.py --hw 576x960 --batch 8 --steps 5     (global batch = 8 * world)
    python tools/train_bench.py --network MaskFlownet --hw 320x768 --batch 4 --steps 10 [--fix-head] [--deterministic]

--network MaskFlownet trains the cascade (the reference's cascade training shape is 320x768, batch 4); --fix-head freezes
its MaskFlownet-S head and gives Adam only the trainable parameters, as PipelineFlownet.fix_head does.  --deterministic runs
the steps under torch.use_deterministic_algorithms(True) (PipelineFlownet(deterministic=True)): the bit-reproducible
kernels, deterministic cuDNN algorithms, cudnn.benchmark off; CUBLAS_WORKSPACE_CONFIG defaults to :4096:8.

Prints one JSON line: ms/step, pairs/s, time of the hand-written backward kernels (CUDA events) and of the all-reduce.
"""
import argparse, json, os, sys, time
if "--deterministic" in sys.argv:                           # must be set before CUDA initialises
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import _lib, dist as mdist, losses, network


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hw", default="384x512")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--network", choices=("MaskFlownet_S", "MaskFlownet"), default="MaskFlownet_S")
    ap.add_argument("--fix-head", action="store_true", help="freeze the cascade's MaskFlownet-S head (MaskFlownet only)")
    ap.add_argument("--deterministic", action="store_true", help="bit-reproducible steps (torch.use_deterministic_algorithms)")
    a = ap.parse_args()
    if a.fix_head and a.network != "MaskFlownet":
        ap.error("--fix-head needs --network MaskFlownet (only the cascade has a head)")
    H, W = map(int, a.hw.split("x"))
    rank, local, world = mdist.init_from_env("nccl")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = not a.deterministic
    if a.deterministic:
        torch.use_deterministic_algorithms(True)
    torch.manual_seed(0)
    model = (network.MaskFlownet() if a.network == "MaskFlownet" else network.MaskFlownetS()).to(dev).train()
    if a.fix_head:                                          # PipelineFlownet.fix_head (network/MaskFlownet.py:412-414)
        for p in model.MaskFlownet_S.parameters():
            p.requires_grad_(False)
    bucket = mdist.GradBucket(model.parameters())           # skips frozen parameters
    opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-4)     # network/pipeline.py:27
    g = torch.Generator(device=dev).manual_seed(1 + rank)
    im1 = torch.rand(a.batch, 3, H, W, device=dev, generator=g) - 0.5
    im2 = torch.rand(a.batch, 3, H, W, device=dev, generator=g) - 0.5
    flow = torch.randn(a.batch, 2, H, W, device=dev, generator=g) * 3
    mask = torch.ones(a.batch, 1, H, W, device=dev)
    t_ar = []

    def step():
        bucket.zero_()
        preds, _, _ = model(im1, im2)
        loss = losses.multiscale_epe(flow, mask, preds).sum()     # per-sample losses are summed (pipeline.py:112-113)
        loss.backward()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        bucket.allreduce_(global_batch=a.batch * world)           # trainer.step(batch_size) (pipeline.py:114)
        e1.record()
        opt.step()
        t_ar.append((e0, e1))
        return loss

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    if world > 1:
        torch.distributed.barrier()
    t_ar.clear()
    n0 = _lib.launch_count()
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    for _ in range(a.steps):
        loss = step()
    s1.record()
    torch.cuda.synchronize()
    ms = mdist.max_over_ranks(s0.elapsed_time(s1), dev) / a.steps
    ar = sum(x.elapsed_time(y) for x, y in t_ar) / len(t_ar)
    if rank == 0:
        print(json.dumps({"bench": "train_step", "network": a.network, "fix_head": a.fix_head,
                          "deterministic": a.deterministic, "hw": a.hw, "batch_per_gpu": a.batch, "n_gpus": world,
                          "ms_per_step": round(ms, 3), "pairs_per_s": round(a.batch * world / ms * 1e3, 2),
                          "native_launches_per_step": (_lib.launch_count() - n0) // a.steps,
                          "grad_allreduce_ms": round(ar, 4), "grad_bucket_mb": round(bucket.numel * 4 / 1e6, 1),
                          "loss": float(loss)}))
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
