"""Training-step time of DIFFormer (medium/difformer.py, kernel='simple', one head) on the CUDA kernels next to the same step
as torch ops (oracle/difformer_oracle.py on the same GPU): forward, loss, backward, Adam.

    python scripts/bench_difformer.py [--steps 50] [--warmup 10]

Shapes: Actor and Squirrel of medium/run.sh (synthetic graphs and features of their sizes, h=64, 8 layers) and one HBM-bound
arxiv-sized shape (h=256, 2 layers) in fp32 and bf16.  Prints one JSON line per shape, after one line with the GPU's name and
power limit.  The bytes per layer are the algorithmic traffic of the kernel schedule (layer_bytes below),
reported as the time they take at the H100 SXM data-sheet 3.35 TB/s and as that time's share of the measured step (the step also
runs the input and output Linear, the loss and Adam)."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import difformer_oracle as O  # noqa: E402
from sgformer_b200.difformer import DIFFormer  # noqa: E402
from sgformer_b200.loss import nll_loss_from_logits  # noqa: E402
from sgformer_b200.optim import Adam  # noqa: E402

HBM = 3.35e12
SHAPES = [("actor", 7600, 932, 5, 30019, 64, 8, "fp32"), ("actor", 7600, 932, 5, 30019, 64, 8, "bf16"),
          ("squirrel", 5201, 2089, 5, 216933, 64, 8, "fp32"), ("squirrel", 5201, 2089, 5, 216933, 64, 8, "bf16"),
          ("arxiv", 169343, 128, 40, 2315598, 256, 2, "fp32"), ("arxiv", 169343, 128, 40, 2315598, 256, 2, "bf16")]


class Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei}


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return info


def layer_bytes(n, h, e, act_bytes):
    """Algorithmic bytes of one layer's training step, every [N, h] activation moved once per pass that needs it.
    Forward: the Gram pass reads x; the apply GEMM reads x and writes o; the V projection reads x and writes dinv v; the SpMM
    reads the column ids, dinv v and writes y; the row pass reads o, x, y and writes the output.  Backward: the row prologue
    reads dy, o, x, y and writes gnum', dr and dinv c du; x^T gnum' reads x and gnum'; the transposed SpMM reads the ids and
    its operand and writes dv; dv^T x and the column sum read dv and x; the dx GEMM reads gnum', x, dv and dr, and writes dx."""
    row = n * h * act_bytes
    ids = e * 4 + n * 8
    fwd = row + 2 * row + 2 * row + (ids + 2 * row) + 4 * row
    bwd = 7 * row + 2 * row + (ids + 2 * row) + 2 * row + 5 * row
    return fwd + bwd


def time_steps(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def run(name, n, d, c, e, h, nl, prec, steps, warmup):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(n, d, generator=g).cuda()
    ei = torch.randint(0, n, (2, e), generator=g).cuda()
    y = torch.randint(0, c, (n,), generator=g).cuda()
    torch.manual_seed(0)
    model = DIFFormer(d, h, c, num_layers=nl, alpha=0.5, dropout=0.5).cuda().set_precision(prec)
    opt = Adam(model.parameters(), lr=1e-3, weight_decay=5e-4)
    data = Data(x, ei)

    def kstep():
        opt.zero_grad(set_to_none=True)
        model.train()
        nll_loss_from_logits(model(data), y).backward()
        opt.step()

    ms = time_steps(kstep, steps, warmup)
    torch_ms = None
    if prec == "fp32":
        cfg = O.make_config(d, h, c, num_layers=nl, dropout=0.5)
        sd = {k: v.detach().clone().requires_grad_(True) for k, v in model.state_dict().items()}
        topt = torch.optim.Adam(list(sd.values()), lr=1e-3, weight_decay=5e-4)

        def tstep():
            topt.zero_grad(set_to_none=True)
            F.cross_entropy(O.difformer_forward(cfg, sd, x, ei, training=True), y).backward()
            topt.step()

        torch_ms = time_steps(tstep, steps, warmup)
    act = 4 if prec == "fp32" else 2
    lb = layer_bytes(n, h, e, act)
    return dict(shape=name, precision=prec, nodes=n, features=d, edges=e, hidden=h, layers=nl, kernel_ms_per_step=round(ms, 3),
                torch_ms_per_step=None if torch_ms is None else round(torch_ms, 3),
                speedup=None if torch_ms is None else round(torch_ms / ms, 2), layer_bytes=lb,
                layer_bytes_us_at_3_35TBps=round(lb / HBM * 1e6, 2),
                layers_bytes_share_of_step=round(nl * lb / HBM * 1e3 / ms, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--only", default=None, help="run one shape name")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_difformer.py needs a CUDA device")
    print(json.dumps(gpu_info()), flush=True)
    for s in SHAPES:
        if a.only and s[0] != a.only:
            continue
        print(json.dumps(run(*s, a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
