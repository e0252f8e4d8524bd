#!/usr/bin/env python
"""bench.py — nodes/sec of one SGFormer training step (fwd + loss + bwd + Adam) on synthetic graphs of the reference's
shapes (BASELINE.json).  One JSON line on stdout (rank 0).

    python bench.py --gpus 1 --steps 10 --warmup 3                       # ogbn-products-shaped, bf16, full batch (config 3)
    python -m torch.distributed.run --nproc-per-node N ... bench.py --gpus N ...   # rank-local graph partitions + grad allreduce
    python bench.py --impl reference                                     # the reference's CPU path (oracle port) on host cores
    python bench.py --steps 10 --warmup 3 --dump-outputs DIR             # + DIR/*.npy: what the last timed step computed

Timed region: device-timed with CUDA events on the launching stream, barrier + synchronize on both sides, max over
ranks.  `value` has the inputs resident in HBM; `e2e` copies the step's inputs from pinned host memory every step
(through `sgformer_b200.feed.HostFeeder`: step i+1's copy AND the CSR build from its fresh edge_index run on a copy stream
beside step i - still inside the timed region, every step) and reads the loss back.  `roofline` is the CSR SpMM (the dominant kernel): algorithmic
bytes per launch (DESIGN.md §SpMM) / its CUDA-event duration inside the timed steps, against MEASURED_PEAKS.json.

Besides the headline line (BASELINE config 3, dp weak scaling at N > 1) the `extra` block carries the other BASELINE
configurations measured in the same process, each next to its own single-GPU baseline:
    N = 1 : config 2 (ogbn-arxiv-shaped, fp32), config 4 at 1 GPU (Pokec-shaped), config 5 at 1 GPU (papers100M-shaped mini-batches)
    N > 1 : row-sharded strong scaling of the products graph (and of the Pokec graph), papers100M-shaped mini-batches dp
(`--no-extra` skips them).
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

# workload -> (N, d_in, E_stored, classes, hidden, gnn layers, use_init, precision)
WORKLOADS = {
    "products": dict(n=2449029, d=100, e=61859140, c=47, h=256, layers=3, use_init=True, precision="bf16"),
    "arxiv": dict(n=169343, d=128, e=1166243, c=40, h=256, layers=3, use_init=False, precision="fp32"),
    "pokec": dict(n=1632803, d=65, e=30622564, c=2, h=64, layers=2, use_init=True, precision="bf16"),
    "papers-batch": dict(n=400000, d=128, e=430000, c=172, h=256, layers=3, use_init=True, precision="bf16"),
    # ogbn-papers100M-shaped, one GPU's shard of an 8-way node partition (111 M / 8 nodes; 1/8 of a node's ~29.7 neighbours are
    # in the same shard), trained with the random-partition mini-batches of large/main-batch.py (batch 400 k, slides / run.sh)
    "papers100M-minibatch": dict(n=13882494, d=128, e=25700000, c=172, h=256, layers=3, use_init=True, precision="bf16",
                                 batch=400000),
    "tiny": dict(n=20000, d=64, e=200000, c=7, h=64, layers=2, use_init=True, precision="bf16"),
}
CONFIG_OF = {"arxiv": 2, "products": 3, "pokec": 4, "papers100M-minibatch": 5}


def model_kwargs(w):
    # large/run.sh recipes: 1 attention layer (residual, weight, LN; no act), GCN with bn/residual/weight/act
    return dict(trans_num_layers=1, trans_num_heads=1, trans_dropout=0.0, trans_use_bn=True, trans_use_residual=True,
                trans_use_weight=True, trans_use_act=False, gnn_num_layers=w["layers"], gnn_dropout=0.0, gnn_use_weight=True,
                gnn_use_init=w["use_init"], gnn_use_bn=True, gnn_use_residual=True, gnn_use_act=True, use_graph=True,
                graph_weight=0.5, aggregate="add")


def peaks():
    try:
        p = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        return float(p["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    except Exception:
        return 3350.0, "H100 SXM data sheet HBM3 bandwidth (not measured)"


def gpu_info(index):
    """Name and power limit of the measuring GPU: a time means little without them (a card may be capped below 700 W)."""
    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(index)],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return info


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled during the timed region."""
    Q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.proc, self.lines = index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i",
                                          str(self.index), "-lms", "100"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                                         text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return None
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [t.strip() for t in ln.split(",")]
            if len(f) < 6:
                continue
            try:
                sm.append(float(f[0])); mx.append(float(f[1]))
            except ValueError:
                continue
            for nm, v in zip(names, f[2:6]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        if not sm:
            return None
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(mx), "reasons": sorted(reasons), "samples": len(sm)}


DUMP_ROWS = 65536      # logits rows sampled into --dump-outputs (fixed seed): 65536 x 172 classes x 4 B = 45 MB at most
DUMP_MAX_BYTES = 64 << 20


def dump_outputs(path, out, loss, model):
    """Write what the timed step computed in its last call, as DIR/<name>.npy (float32; row indices float64): the loss, the
    logits of a fixed seeded sample of rows (all rows when there are fewer) and every parameter after the optimizer step."""
    import numpy as np
    os.makedirs(path, exist_ok=True)
    n = out.shape[0]
    rows = torch.randperm(n, generator=torch.Generator().manual_seed(0))[:DUMP_ROWS].sort().values
    arrays = {"loss": loss.detach().float().reshape(1).cpu().numpy(),
              "logits_sample": out.detach()[rows.to(out.device)].float().cpu().numpy(),
              "logits_sample_rows": rows.numpy().astype(np.float64)}
    for name, prm in model.named_parameters():
        arrays["param." + name] = prm.detach().float().cpu().numpy()
    total = sum(a.nbytes for a in arrays.values())
    if total > DUMP_MAX_BYTES:
        raise RuntimeError(f"--dump-outputs: {total} bytes exceed {DUMP_MAX_BYTES}")
    for name, a in arrays.items():
        np.save(os.path.join(path, name + ".npy"), a)


def spmm_algorithmic_bytes(n, nnz, h, b):
    """SURVEY.md §8d: nnz*4 (int32 col) + (n+1)*8 (int64 rowptr) + nnz*h*b (gathered rows) + n*h*b (output)."""
    return nnz * 4 + (n + 1) * 8 + nnz * h * b + n * h * b


# ------------------------------------------------------------------------------------------------
# reference arm / cpu_baseline: the oracle port on the host cores, bounded sample
# ------------------------------------------------------------------------------------------------
_best_threads = {}


def _cpu_step_fn(w, n, e):
    from oracle import sgformer_oracle as O
    from sgformer_b200.synth import make_graph
    kw = model_kwargs(w)
    cfg = O.make_config("large", w["d"], w["h"], w["c"], **kw)
    sd = O.init_state_dict(cfg, seed=0)
    ei = make_graph(n, e, seed=0)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(n, w["d"], generator=g)
    y = torch.randint(0, w["c"], (n,), generator=g)

    def step():
        sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else v.clone())
               for k, v in sd.items()}
        out = O.sgformer_forward(cfg, sdg, x, ei, training=True)
        torch.nn.functional.nll_loss(torch.log_softmax(out, 1), y).backward()

    return step, ei.shape[1]


def _timed_cpu(step, repeats):
    best = float("inf")
    for _ in range(max(1, repeats)):
        t0 = time.perf_counter()
        step()
        best = min(best, time.perf_counter() - t0)
    return best


def pick_threads(w):
    """The oracle's speed on the box's host cores depends strongly on the thread count (r1: 2.3 k vs 13.3 k nodes/s for the same
    code under two launchers): sweep 8..cpu_count on a small sample and keep the fastest."""
    key = (w["h"], w["d"])
    if key in _best_threads:
        return _best_threads[key]
    ncpu = os.cpu_count() or 1
    cands = sorted({t for t in (8, 16, 32, 64, 128, ncpu) if t <= ncpu} or {ncpu})
    step, _ = _cpu_step_fn(w, 12000, max(1000, int(w["e"] * 12000 / w["n"])))
    res = {}
    for t in cands:
        torch.set_num_threads(t)
        step()
        res[t] = _timed_cpu(step, 1)
    best = min(res, key=res.get)
    _best_threads[key] = (best, {str(k): round(12000 / v) for k, v in res.items()})
    return _best_threads[key]


def cpu_reference(w, budget_nodes=60000, repeats=1, full=False):
    threads, sweep = pick_threads(w)
    torch.set_num_threads(threads)
    frac = 1.0 if full else min(1.0, budget_nodes / w["n"])
    n = max(1000, int(w["n"] * frac))
    e = max(1000, int(w["e"] * frac))          # same average degree as the full workload
    step, nnz = _cpu_step_fn(w, n, e)
    best = _timed_cpu(step, repeats)
    what = "the FULL workload" if frac == 1.0 else f"a {n}-node / {nnz}-edge subsample with the workload's mean degree"
    return dict(value=n / best, unit="nodes/s", cores=threads, kind="port",
                sample=f"oracle/sgformer_oracle.py (torch-CPU restatement of large/ours.py; the reference's own ours.py needs "
                       f"torch_sparse/torch_geometric, absent on the GPU box) train-mode fwd+bwd on {what}, fp32, {threads} threads "
                       f"(fastest of the sweep {sweep} nodes/s), best of {max(1, repeats)}", seconds=best, nodes=n,
                thread_sweep_nodes_per_s=sweep, same_config=frac == 1.0)


def run_reference(args, w, wname):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    t_all = time.perf_counter()
    vals = []
    for _ in range(args.warmup):
        cpu_reference(w, budget_nodes=10000)
    res = None
    for _ in range(max(1, args.steps)):
        res = cpu_reference(w, budget_nodes=args.ref_nodes)
        vals.append(res["seconds"])
        if time.perf_counter() - t_all > 200:
            break
    sec = statistics.mean(vals)
    value = res["nodes"] / sec
    line = {"impl": "reference", "metric": "nodes/sec fwd+bwd", "value": value, "unit": "nodes/s", "n_gpus": args.gpus,
            "steps": len(vals), "warmup": args.warmup, "ms_per_step": sec * 1e3, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": f"ogbn-{wname}-shaped synthetic, full batch", "sample_nodes": res["nodes"], "hidden": w["h"],
                       "gnn_layers": w["layers"], "cpu_threads": res["cores"], "kind": "port",
                       "thread_sweep_nodes_per_s": res["thread_sweep_nodes_per_s"]},
            "cpu_baseline": {k: res[k] for k in ("unit", "cores", "kind", "sample")} | {"value": value},
            "e2e": {"value": value, "unit": "nodes/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line), flush=True)


# ------------------------------------------------------------------------------------------------
# ours
# ------------------------------------------------------------------------------------------------
class Ctx:
    """Process-wide distributed context of one bench invocation."""

    def __init__(self):
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local = int(os.environ.get("LOCAL_RANK", "0"))
        if not torch.cuda.is_available():
            raise RuntimeError("bench.py --impl ours needs a CUDA device (no CPU fallback)")
        torch.cuda.set_device(self.local)
        self.dev = torch.device("cuda", self.local)
        self.dist = None
        if self.world > 1:
            import torch.distributed as dist
            import datetime
            dist.init_process_group("nccl", device_id=self.dev,
                                    timeout=datetime.timedelta(seconds=int(os.environ.get("SGF_BENCH_INIT_TIMEOUT", "300"))))
            self.dist = dist

    def barrier(self):
        if self.dist is not None:
            self.dist.barrier()

    def timed(self, fn, steps, world):
        """CUDA events around `steps` calls, barrier + synchronize on both sides, max over the `world` participating ranks."""
        if world > 1:
            self.dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        if world > 1:
            self.dist.barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=self.dev)
        if world > 1:
            self.dist.all_reduce(ms, op=self.dist.ReduceOp.MAX)
        return ms.item() / steps


def _optimizer(model, graph_capturable=True):
    from sgformer_b200.optim import Adam
    return Adam([{"params": model.params1, "weight_decay": 0.0}, {"params": model.params2, "weight_decay": 0.0}], lr=1e-3)


def run_full_batch(ctx, wname, w, parallel, steps, warmup, want_e2e=False, want_roofline=False, use_graph=True, rmat=False,
                   solo=False, sample_clocks=False, dump_dir=None):
    """One full-batch measurement.  parallel: 'single' | 'dp' | 'rows'.  solo=True: rank 0 alone (a single-GPU baseline taken
    inside a multi-rank job; the other ranks return None and wait at the caller's barrier).  dump_dir: rank 0 writes the
    outputs of the last timed step there (dump_outputs)."""
    from sgformer_b200 import kernels as K
    from sgformer_b200 import large as L
    from sgformer_b200.graph import clear_cache, get_graph
    from sgformer_b200.loss import nll_loss_from_logits
    from sgformer_b200.synth import make_graph, make_rmat_graph
    gen = make_rmat_graph if rmat else make_graph
    dist, dev, rank = ctx.dist, ctx.dev, ctx.rank
    world = 1 if (solo or parallel == "single") else ctx.world
    if solo and rank != 0:
        return None
    torch.manual_seed(1234)
    n, d, c, h = w["n"], w["d"], w["c"], w["h"]
    rows_mode = world > 1 and parallel == "rows"
    comm = None
    if rows_mode:
        # one global graph (same seed everywhere); every rank keeps its row block of x / y and builds its CSR row shard
        from sgformer_b200.dist import Comm
        comm = Comm(dist.group.WORLD, n)
        r0, r1 = comm.rows
        ei = gen(n, w["e"], seed=100, device=dev)
        g = torch.Generator(device=dev).manual_seed(7)
        x = torch.randn(n, d, generator=g, device=dev)[r0:r1].contiguous()
        y = torch.randint(0, c, (n,), generator=g, device=dev)[r0:r1].contiguous()
    else:
        # rank-local graph partition of the named shape (same shape on every rank, different seed): weak scaling
        sr = rank if world > 1 else 0
        ei = gen(n, w["e"], seed=100 + sr, device=dev)
        g = torch.Generator(device=dev).manual_seed(7 + sr)
        x = torch.randn(n, d, generator=g, device=dev)
        y = torch.randint(0, c, (n,), generator=g, device=dev)
    model = L.SGFormer(d, h, c, **model_kwargs(w)).to(dev).set_precision(w["precision"])
    if rows_mode:
        model.set_row_sharding(comm)
    if world > 1:
        for p in model.parameters():
            dist.broadcast(p.data, 0)
    opt = _optimizer(model)
    model.train()
    params = [p for p in model.parameters()]

    def allreduce_grads():
        if world == 1 or rows_mode:      # row-sharded: the backward already all-reduces the gradients (C5)
            return
        flat = torch.cat([p.grad.reshape(-1) for p in params if p.grad is not None])
        dist.all_reduce(flat)
        flat.div_(world)
        o = 0
        for p in params:
            if p.grad is not None:
                k = p.grad.numel()
                p.grad.copy_(flat[o:o + k].view_as(p.grad))
                o += k

    last = {}      # logits and loss of the latest step (inside a captured graph: the graph's output buffers)

    def step(xd, eid, yd):
        opt.zero_grad(set_to_none=True)
        out = model(xd, eid)
        loss = nll_loss_from_logits(out, yd, None, float(n))   # mean over the (global) node count; fused fwd+grad kernel
        loss.backward()
        allreduce_grads()
        opt.step()
        last.update(out=out.detach(), loss=loss.detach())     # detached: must not keep the step's autograd graph alive
        return loss

    for _ in range(warmup):
        step(x, ei, y)
    # The whole step (zero_grad .. Adam) is a static kernel schedule: capture it once in a CUDA graph and replay it (falls back
    # to eager launches if capture is not possible).  Multi-GPU steps are captured too - NCCL collectives, the copy-engine pushes
    # of the halo exchange and their flag kernels are all graph nodes - and every rank replays only if every rank captured.
    run_step = lambda: step(x, ei, y)  # noqa: E731
    used_graph = False
    if use_graph and (world == 1 or os.environ.get("SGF_BENCH_MULTI_GRAPH", "1") == "1"):
        cg = None
        try:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                step(x, ei, y)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            cg = torch.cuda.CUDAGraph()
            with torch.cuda.graph(cg):
                step(x, ei, y)
            captured = dict(last)
        except Exception as exc:  # pragma: no cover
            print(f"[bench] CUDA graph capture failed ({type(exc).__name__}: {exc}); running eagerly", file=sys.stderr)
            cg = None
        torch.cuda.synchronize()
        ok = torch.tensor([1 if cg is not None else 0], device=dev)
        if world > 1:
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if int(ok.item()) == 1:
            cg.replay()
            torch.cuda.synchronize()
            run_step = cg.replay
            used_graph = True
    graph = get_graph(ei, n, 0, rows=comm.rows, col_rot=comm.col_rot) if rows_mode else get_graph(ei, n, 0)
    nnz = graph.nnz
    sampler = ClockSampler(ctx.local) if (rank == 0 and sample_clocks) else None
    if sampler:
        sampler.start()
    l0 = K.launch_count()
    ev = []
    if used_graph:
        # kernels replayed from the graph are not re-issued through the C-ABI: count one eager step for gpu_launches
        step(x, ei, y)
        per_step = K.launch_count() - l0
        ms_step = ctx.timed(run_step, steps, world)
        if dump_dir and rank == 0:
            dump_outputs(dump_dir, captured["out"], captured["loss"], model)
        launches = per_step * steps
        if want_roofline:
            # SpMM launch durations for the roofline: a few eager steps with CUDA events around each SpMM launch
            K.spmm_events = []
            ctx.timed(lambda: step(x, ei, y), 2, world)
            ev, K.spmm_events = K.spmm_events, None
    else:
        K.spmm_events = [] if want_roofline else None
        ms_step = ctx.timed(run_step, steps, world)
        if dump_dir and rank == 0:
            dump_outputs(dump_dir, last["out"], last["loss"], model)
        launches = K.launch_count() - l0
        ev, K.spmm_events = (K.spmm_events or []), None
    clocks = sampler.stop() if sampler else None
    spmm_ms = [a.elapsed_time(b) for a, b in ev]
    total_nodes = n if (rows_mode or world == 1) else n * world
    res = dict(ms_per_step=ms_step, value=total_nodes / (ms_step * 1e-3), launches=launches, used_graph=used_graph, nnz=nnz,
               clocks=clocks, world=world, rows_mode=rows_mode, n=n, graph_rows=graph.rowptr.numel() - 1, e2e=None, roofline=None)

    # end to end: inputs come from pinned host memory every step, loss is read back
    if want_e2e:
        xh, eih, yh = x.cpu().pin_memory(), ei.cpu().pin_memory(), y.cpu().pin_memory()
        h2d = xh.numel() * xh.element_size() + eih.numel() * eih.element_size() + yh.numel() * yh.element_size()
        # public API path: HostFeeder stages step i+1's inputs on a copy stream while step i computes (one full copy of
        # x / edge_index / y from pinned memory per step inside the timed region) and builds the CSR of the freshly copied
        # edge_index behind the copy on the same stream (model.prepare_graph); the loss is read back every step
        from sgformer_b200.feed import HostFeeder
        feeder = HostFeeder(dev, prepare=(lambda xd, eid, yd: model.prepare_graph(eid, xd.shape[0]))
                            if os.environ.get("SGF_BENCH_PREPARE", "1") == "1" and not rows_mode else None)
        feeder.submit((xh, eih, yh))

        def e2e_step():
            xd, eid, yd = feeder.get()
            loss = step(xd, eid, yd)             # enqueued first: the GPU works on it while the host sits in the next submit
            feeder.submit((xh, eih, yh))
            return loss.item()

        e2e_step()
        ms_e2e = ctx.timed(e2e_step, max(2, min(steps, 5)), world)
        res["e2e"] = {"value": total_nodes / (ms_e2e * 1e-3), "unit": "nodes/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4,
                      "ms_per_step": ms_e2e}
        del feeder, xh, eih, yh
    if want_roofline and spmm_ms and rank == 0:
        b = 2 if w["precision"] == "bf16" else 4
        alg = spmm_algorithmic_bytes(res["graph_rows"], nnz, h, b)
        peak, peak_src = peaks()
        avg_ms = statistics.mean(spmm_ms)
        achieved = alg / (avg_ms * 1e-3) / 1e9
        timed_steps = 2 if used_graph else steps
        res["roofline"] = {"kernel": "spmm_rows_kernel (CSR SpMM fwd + transposed bwd)", "bound": "hbm", "achieved": achieved,
                           "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                           # dram__bytes of this exact launch are only known from a profiler capture: not measured live
                           "traffic": None, "peak_source": peak_src, "algorithmic_bytes_per_launch": alg,
                           "avg_launch_ms": avg_ms, "launches_timed": len(spmm_ms),
                           "share_of_step": avg_ms * (len(spmm_ms) / timed_steps) / ms_step}
    del model, opt, x, y, ei, graph, params
    clear_cache()
    gc.collect()
    torch.cuda.empty_cache()
    return res


def run_minibatch(ctx, w, steps, warmup, solo=False, dump_dir=None):
    """papers100M-shaped random-partition mini-batches (large/main-batch.py:130-151) kept on the device: CSR built once, per step a
    random batch -> Graph.subset (K9 on the CSR) -> feature gather -> fwd/bwd -> (grad all-reduce) -> Adam."""
    from sgformer_b200 import kernels as K
    from sgformer_b200 import large as L
    from sgformer_b200.graph import Graph, clear_cache
    from sgformer_b200.loss import nll_loss_from_logits
    from sgformer_b200.minibatch import RandomPartitionSampler
    from sgformer_b200.synth import make_graph
    dist, dev, rank = ctx.dist, ctx.dev, ctx.rank
    world = 1 if solo else ctx.world
    if solo and rank != 0:
        return None
    torch.manual_seed(1234)
    n, d, c, h = w["n"], w["d"], w["c"], w["h"]
    sr = rank if world > 1 else 0
    ei = make_graph(n, w["e"], seed=100 + sr, device=dev)
    g = torch.Generator(device=dev).manual_seed(7 + sr)
    x = torch.randn(n, d, generator=g, device=dev)
    y = torch.randint(0, c, (n,), generator=g, device=dev)
    model = L.SGFormer(d, h, c, **model_kwargs(w)).to(dev).set_precision(w["precision"])
    if world > 1:
        for p in model.parameters():
            dist.broadcast(p.data, 0)
    opt = _optimizer(model)
    model.train()
    params = [p for p in model.parameters()]
    full = Graph(ei, n)
    bsz = w["batch"]
    cap = int(bsz * (2.0 * w["e"] / n * bsz / n + 1.0) * 1.5) + 1024     # induced nnz bound: no per-batch device sync
    sampler = RandomPartitionSampler(full, x, y, bsz, capacity=cap, generator=torch.Generator(device=dev).manual_seed(11 + sr))
    batches = iter(())
    last = {}

    def mb_step():
        nonlocal batches
        mb = next(batches, None)
        if mb is None or mb.idx.numel() < bsz:      # new epoch (skip the ragged last batch: fixed work per step)
            batches = iter(sampler)
            mb = next(batches)
        opt.zero_grad(set_to_none=True)
        out = model(mb)
        loss = nll_loss_from_logits(out, mb.labels, None, float(bsz))
        loss.backward()
        if world > 1:
            flat = torch.cat([p.grad.reshape(-1) for p in params if p.grad is not None])
            dist.all_reduce(flat)
            flat.div_(world)
            o = 0
            for p in params:
                if p.grad is not None:
                    k = p.grad.numel()
                    p.grad.copy_(flat[o:o + k].view_as(p.grad))
                    o += k
        opt.step()
        last.update(out=out.detach(), loss=loss.detach())     # detached: must not keep the step's autograd graph alive
        return loss

    for _ in range(warmup):
        mb_step()
    l0 = K.launch_count()
    ms_step = ctx.timed(mb_step, steps, world)
    if dump_dir and rank == 0:
        dump_outputs(dump_dir, last["out"], last["loss"], model)
    launches = K.launch_count() - l0
    sampler.check()         # a batch whose induced subgraph exceeded `cap` would have been truncated: fail loudly
    res = dict(ms_per_step=ms_step, value=bsz * world / (ms_step * 1e-3), launches=launches, nnz=full.nnz, world=world, n=n, batch=bsz)
    del model, opt, x, y, ei, full, sampler, params
    clear_cache()
    gc.collect()
    torch.cuda.empty_cache()
    return res


def _brief(r, **more):
    if r is None:
        return None
    out = {"ms_per_step": round(r["ms_per_step"], 4), "nodes_per_s": r["value"], "n_gpus": r["world"],
           "cuda_graph": r.get("used_graph", False)}
    out.update(more)
    return out


def extras(ctx, args):
    """The BASELINE configurations the headline line does not cover, each with its own single-GPU baseline from this process."""
    world, rank = ctx.world, ctx.rank
    st, wu = max(3, min(args.steps, 10)), 3
    out = {}
    t_begin = time.perf_counter()
    budget = float(os.environ.get("SGF_BENCH_EXTRA_BUDGET", "330"))      # seconds: later items are skipped, never cut short

    def guard(name, fn):
        # every rank takes the same decision (rank 0's clock)
        over = torch.tensor([1 if time.perf_counter() - t_begin > budget else 0], device=ctx.dev)
        if ctx.dist is not None:
            ctx.dist.broadcast(over, 0)
        if int(over.item()):
            out[name] = {"skipped": f"extra-measurement time budget of {budget:.0f} s used up"}
            return
        try:
            out[name] = fn()
        except Exception as exc:  # one failing extra must not take the headline line down
            out[name] = {"error": f"{type(exc).__name__}: {exc}"[:300]}
            torch.cuda.synchronize()
        ctx.barrier()

    if world == 1:
        guard("config2_arxiv_fp32", lambda: _brief(run_full_batch(ctx, "arxiv", dict(WORKLOADS["arxiv"]), "single", 2 * st, wu),
                                                   workload="ogbn-arxiv-shaped synthetic (169 343 nodes, 128-d, 1.17 M edges), full batch, fp32 (bf16x3 tensor-core products)"))
        guard("config4_pokec_1gpu", lambda: _brief(run_full_batch(ctx, "pokec", dict(WORKLOADS["pokec"]), "single", 2 * st, wu),
                                                   workload="Pokec-shaped synthetic (1.63 M nodes, 65-d, 30.6 M edges), full batch, bf16"))
        guard("config5_papers100M_minibatch_1gpu",
              lambda: _brief(run_minibatch(ctx, dict(WORKLOADS["papers100M-minibatch"]), 2 * st, wu),
                             workload="papers100M-shaped shard (13.9 M nodes), random-partition mini-batches of 400 k nodes, bf16"))
        return out

    def strong(name, wname, label):
        w = dict(WORKLOADS[wname])

        def fn():
            try:
                base = run_full_batch(ctx, wname, w, "single", st, wu, solo=True)      # rank 0 alone; the others wait below
            except Exception as exc:      # keep the ranks' barrier sequence aligned whatever happens to the baseline
                print(f"[bench] single-GPU baseline of {wname} failed: {exc}", file=sys.stderr)
                base = None
                torch.cuda.synchronize()
            ctx.barrier()
            b = torch.tensor([base["ms_per_step"] if base else float("nan")], device=ctx.dev)
            ctx.dist.broadcast(b, 0)
            r = run_full_batch(ctx, wname, w, "rows", st, wu)
            return _brief(r, workload=label, parallelism=f"rows{world}: one graph, nodes row-sharded (C1-C5)", scaling="strong",
                          baseline_1gpu_ms=round(b.item(), 4), speedup_vs_1gpu=b.item() / r["ms_per_step"])
        guard(name, fn)

    strong("config3_products_rows", "products", "ogbn-products-shaped synthetic, ONE graph row-sharded over the GPUs, bf16")
    strong("config4_pokec_rows", "pokec", "Pokec-shaped synthetic, ONE graph row-sharded over the GPUs, bf16 (BASELINE config 4: 2 and 4 GPUs)")

    def mb():
        w = dict(WORKLOADS["papers100M-minibatch"])
        try:
            base = run_minibatch(ctx, w, st, wu, solo=True)
        except Exception as exc:
            print(f"[bench] single-GPU mini-batch baseline failed: {exc}", file=sys.stderr)
            base = None
            torch.cuda.synchronize()
        ctx.barrier()
        b = torch.tensor([base["value"] if base else float("nan")], device=ctx.dev, dtype=torch.float64)
        ctx.dist.broadcast(b, 0)
        r = run_minibatch(ctx, w, st, wu)
        return _brief(r, workload="papers100M-shaped: per-GPU node shard (13.9 M nodes), random-partition mini-batches of 400 k nodes "
                      "per GPU (large/main-batch.py), replicated model, NCCL grad all-reduce", scaling="weak",
                      baseline_1gpu_nodes_per_s=b.item(), speedup_vs_1gpu=r["value"] / b.item())
    guard("config5_papers100M_minibatch_dp", mb)
    return out


def extras_in_children(ctx, args):
    """N > 1: the extra measurements run in a second set of processes (one child per rank, its own rendezvous port and NCCL
    communicator, the same GPU) so that whatever happens to them - a failed collective, a trapped kernel - cannot take the headline
    line down; the parents idle meanwhile with their caches released."""
    gc.collect()
    torch.cuda.empty_cache()
    env = dict(os.environ)
    env["MASTER_PORT"] = str(int(os.environ.get("MASTER_PORT", "29500")) + 23)
    for k in list(env):          # without torchrun's agent store the children's rank 0 hosts its own TCPStore on the new port
        if k.startswith("TORCHELASTIC_"):
            env.pop(k)
    env["SGF_BENCH_INIT_TIMEOUT"] = "240"
    cmd = [sys.executable, os.path.abspath(__file__), "--extras-child", "--gpus", str(args.gpus), "--steps", str(args.steps),
           "--warmup", str(args.warmup)]
    out = None
    try:
        r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=720)
        for ln in r.stdout.splitlines():
            if ln.startswith("EXTRAS_JSON "):
                out = json.loads(ln[len("EXTRAS_JSON "):])
        if out is None and ctx.rank == 0:
            out = {"error": f"extras child exited with {r.returncode}: " + (r.stderr.strip().splitlines() or [""])[-1][:300]}
    except Exception as exc:
        if ctx.rank == 0:
            out = {"error": f"{type(exc).__name__}: {exc}"[:300]}
    ctx.barrier()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default=os.environ.get("SGF_BENCH_WORKLOAD", "products"), choices=sorted(WORKLOADS))
    ap.add_argument("--precision", default=None, choices=[None, "bf16", "fp32"])
    ap.add_argument("--ref-nodes", type=int, default=60000)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-extra", action="store_true", help="skip the `extra` block (the other BASELINE configurations)")
    ap.add_argument("--extras-child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--rmat", action="store_true", help="power-law R-MAT edges instead of uniform (secondary, not graded)")
    ap.add_argument("--no-graph", action="store_true", help="do not capture the training step in a CUDA graph")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps write what the last one computed (loss, sampled logits, updated parameters) "
                         "as DIR/<name>.npy")
    ap.add_argument("--parallel", default="dp", choices=["dp", "rows"],
                    help="N>1: 'dp' = rank-local graph partitions + gradient all-reduce (weak scaling); 'rows' = ONE graph, "
                         "nodes row-sharded, K^T V / BN all-reduces + SpMM operand all-gather (strong scaling)")
    args = ap.parse_args()
    w = dict(WORKLOADS[args.workload])
    if args.precision:
        w["precision"] = args.precision
    if args.impl == "reference":
        return run_reference(args, w, args.workload)
    if args.warmup < 3:
        args.warmup = 3
    ctx = Ctx()
    rank, world = ctx.rank, ctx.world
    n, d, c, h = w["n"], w["d"], w["c"], w["h"]
    if args.extras_child:
        out = extras(ctx, args)
        if rank == 0:
            print("EXTRAS_JSON " + json.dumps(out), flush=True)
        if world > 1:
            ctx.dist.destroy_process_group()
        return

    if "batch" in w:
        r = run_minibatch(ctx, w, args.steps, args.warmup, dump_dir=args.dump_outputs)
        if rank == 0:
            line = {"metric": "nodes/sec fwd+bwd", "value": r["value"], "unit": "nodes/s", "n_gpus": world,
                    "steps": args.steps, "warmup": args.warmup, "ms_per_step": r["ms_per_step"], "higher_is_better": True,
                    "scaling": "weak", "vs_baseline": None, "dtype": w["precision"], "data": "synthetic",
                    "config": {"workload": "ogbn-papers100M-shaped, random-partition mini-batches (large/main-batch.py)",
                               "batch_nodes_per_gpu": r["batch"], "shard_nodes_per_gpu": n, "shard_nnz": r["nnz"], "in_features": d,
                               "hidden": h, "classes": c, "gnn_layers": w["layers"], "gnn_use_init": True,
                               "parallelism": "single GPU" if world == 1 else
                               f"dp{world}: rank-local node shards, replicated model, NCCL grad allreduce",
                               "step": "sample batch + Graph.subset (K9 on CSR) + feature gather + fwd + fused loss + bwd + Adam",
                               "cuda_graph": False},
                    "e2e": None, "gpu_launches": r["launches"], "clocks": None, "roofline": None, "cpu_baseline": None,
                    "gpu": gpu_info(ctx.local)}
            print(json.dumps(line), flush=True)
        if world > 1:
            ctx.dist.destroy_process_group()
        return

    par = "single" if world == 1 else args.parallel
    r = run_full_batch(ctx, args.workload, w, par, args.steps, args.warmup, want_e2e=not args.no_e2e, want_roofline=True,
                       use_graph=not args.no_graph, rmat=args.rmat, sample_clocks=True, dump_dir=args.dump_outputs)
    ctx.barrier()
    extra = None
    if not args.no_extra and args.workload == "products" and not args.rmat:
        extra = extras(ctx, args) if world == 1 else extras_in_children(ctx, args)
    if rank != 0:
        if world > 1:
            ctx.dist.destroy_process_group()
        return
    cpu = None
    if not args.no_cpu_baseline:
        cpu = cpu_reference(w, budget_nodes=args.ref_nodes)
        cpu = {k: cpu[k] for k in ("value", "unit", "cores", "kind", "sample")}
        if extra is not None and world == 1 and "config2_arxiv_fp32" in extra and "error" not in (extra["config2_arxiv_fp32"] or {}):
            # config 2 fits the host in seconds: the SAME configuration on both arms (full graph, fp32)
            full = cpu_reference(dict(WORKLOADS["arxiv"]), full=True)
            extra["config2_arxiv_fp32"]["cpu_same_config"] = {k: full[k] for k in ("value", "unit", "cores", "kind", "sample", "seconds")}
            extra["config2_arxiv_fp32"]["gpu_over_cpu_same_config"] = extra["config2_arxiv_fp32"]["nodes_per_s"] / full["value"]
    rows_mode = r["rows_mode"]
    line = {"metric": "nodes/sec fwd+bwd", "value": r["value"], "unit": "nodes/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": r["ms_per_step"], "higher_is_better": True,
            "scaling": "strong" if rows_mode else "weak", "vs_baseline": None,
            "dtype": w["precision"], "data": "synthetic",
            "config": {"workload": f"ogbn-{args.workload}-shaped synthetic, full batch" if args.workload != "papers-batch"
                       else "papers100M-shaped mini-batch (400k nodes)", "baseline_config": CONFIG_OF.get(args.workload),
                       "nodes_per_gpu": n, "nnz_per_gpu": r["nnz"],
                       "in_features": d, "hidden": h, "classes": c, "gnn_layers": w["layers"], "gnn_use_init": w["use_init"],
                       "attn_layers": 1, "parallelism": "single GPU" if world == 1 else
                       (f"rows{world}: one graph, nodes row-sharded; NCCL all-reduce of x^T x/x^T 1 (attention) + BN sums + grads, "
                        f"all-gather of the SpMM operand rows" if rows_mode else
                        f"dp{world}: rank-local graph partitions, replicated model, NCCL grad allreduce"),
                       "step": "zero_grad + forward + fused log_softmax/NLL (sgf_softmax_nll) + backward + fused two-group Adam "
                               "(sgf_adam_step)",
                       "cuda_graph": r["used_graph"],
                       "edges": "rmat(.57,.19,.19)" if args.rmat else "uniform",
                       "l2": "inputs (>= 1 GB of activations per pass) exceed the 50 MB L2; no explicit flush"},
            "e2e": r["e2e"], "gpu_launches": r["launches"], "clocks": r["clocks"], "roofline": r["roofline"], "cpu_baseline": cpu,
            "gpu": gpu_info(ctx.local),
            "extra": extra}
    print(json.dumps(line), flush=True)
    if world > 1:
        ctx.dist.destroy_process_group()


if __name__ == "__main__":
    main()
