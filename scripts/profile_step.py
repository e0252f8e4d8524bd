#!/usr/bin/env python
"""Per-kernel attribution of one eager training step of the bench workload (default: products-shaped, bf16, 1 GPU).

Builds the model exactly as bench.py does (same seeds, `model_kwargs`, optimizer), warms it up, and runs one eager step
under torch.profiler with CUDA activities.  Every public function of `sgformer_b200.kernels` is wrapped in a
record_function range named after its call site (caller function and line), and the algorithmic bytes of the call are
computed from its tensor arguments and results: every distinct tensor read or written once, an accumulated output
read and written, and the SpMM's gather as nnz rows of the operand (bench.spmm_algorithmic_bytes).  A kernel in the
trace belongs to the innermost range around its launch.  Prints one row per call site (device time, bytes, fraction of
the HBM bandwidth), the launch count and the sum of the gaps between consecutive GPU activities, and writes the
Chrome trace and the table as JSON under --out.

    python scripts/profile_step.py [--workload products] [--warmup 3] [--out DIR]
"""
import argparse
import collections
import functools
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from sgformer_b200 import kernels as K  # noqa: E402

# helpers of kernels.py that launch nothing themselves (their inner launches are attributed to the wrapped callee)
_NOT_WRAPPED = {"lib", "dcode", "ceil_to", "alloc_act", "new_like", "operand_from_bf16", "as_operand", "stats_fusable",
                "operand_memo_begin", "operand_memo_clear", "dropout_epoch", "launch_count", "heavy_rows"}


def _collect(obj, out):
    if isinstance(obj, torch.Tensor):
        out.append(obj)
    elif isinstance(obj, K.Operand):
        out.append(obj.data)
    elif isinstance(obj, (list, tuple)):
        for o in obj:
            _collect(o, out)
    elif isinstance(obj, dict):
        for o in obj.values():
            _collect(o, out)


def _nbytes(t):
    return t.numel() * t.element_size()


def call_bytes(name, args, kwargs, result):
    """Algorithmic bytes of one kernels.py call (see the module docstring)."""
    if name == "spmm":
        rowptr, col, _, x = args[:4]
        n = rowptr.numel() - 1
        return bench.spmm_algorithmic_bytes(n, col.numel(), x.shape[1], x.element_size())
    ts = []
    _collect(args, ts)
    _collect(kwargs, ts)
    _collect(result, ts)
    seen, total = set(), 0
    for t in ts:
        if not t.is_cuda:
            continue
        key = (t.data_ptr(), _nbytes(t))
        if key not in seen:
            seen.add(key)
            total += key[1]
    if kwargs.get("dres_accumulate") and isinstance(kwargs.get("dres"), torch.Tensor):
        total += _nbytes(kwargs["dres"])
    if name == "gemm_nt" and kwargs.get("accumulate"):
        total += _nbytes(args[4] if len(args) > 4 else kwargs["out"])
    return total


def _site():
    """First frame outside kernels.py and this script: 'module.function:line'."""
    f = sys._getframe(2)
    here = os.path.abspath(__file__)
    while f is not None and (f.f_code.co_filename == K.__file__ or os.path.abspath(f.f_code.co_filename) == here):
        f = f.f_back
    if f is None:
        return "?"
    mod = os.path.splitext(os.path.basename(f.f_code.co_filename))[0]
    return f"{mod}.{f.f_code.co_name}:{f.f_lineno}"


CALLS = []          # (label, site, bytes) per wrapped call, in call order; the record_function range is named "sgf#<index>"


def wrap_kernels():
    for name, fn in list(vars(K).items()):
        if not callable(fn) or name.startswith("_") or name in _NOT_WRAPPED or getattr(fn, "__module__", None) != K.__name__:
            continue
        if isinstance(fn, type):
            continue

        def make(name, fn):
            @functools.wraps(fn)
            def w(*args, **kwargs):
                idx = len(CALLS)
                CALLS.append([name, _site(), 0])
                with torch.profiler.record_function(f"sgf#{idx}"):
                    res = fn(*args, **kwargs)
                CALLS[idx][2] = call_bytes(name, args, kwargs, res)
                return res
            return w
        setattr(K, name, make(name, fn))


def short_kernel(name):
    s = name.split("(")[0]
    if s.startswith("void "):
        s = s[5:]
    return s.replace("sgf::", "").replace("__nv_bfloat16", "bf16")


def attribute(trace_path):
    """-> (rows keyed by call site, GPU activities sorted by start) from a Chrome trace written by torch.profiler."""
    with open(trace_path) as fh:
        ev = json.load(fh)["traceEvents"]
    runtime = {}                                            # correlation -> (tid, ts) of the launching API call
    ranges = collections.defaultdict(list)                  # tid -> [(ts, end, index)]
    gpu = []
    for e in ev:
        cat, args = e.get("cat", ""), e.get("args", {}) or {}
        if cat in ("cuda_runtime", "cuda_driver") and "correlation" in args:
            runtime[args["correlation"]] = (e.get("tid"), e["ts"])
        elif cat == "user_annotation" and str(e.get("name", "")).startswith("sgf#"):
            ranges[e.get("tid")].append((e["ts"], e["ts"] + e.get("dur", 0), int(e["name"][4:])))
        elif cat in ("kernel", "gpu_memset", "gpu_memcpy"):
            gpu.append(e)
    gpu.sort(key=lambda e: e["ts"])
    rows = collections.OrderedDict()
    for e in gpu:
        if e["cat"] != "kernel":
            continue
        corr = (e.get("args", {}) or {}).get("correlation")
        idx = None
        if corr in runtime:
            tid, t = runtime[corr]
            best = None
            for (t0, t1, i) in ranges.get(tid, ()):
                if t0 <= t <= t1 and (best is None or t0 >= best[0]):
                    best = (t0, i)
            idx = best[1] if best else None
        if idx is None:
            key, label = "(launched outside sgformer_b200.kernels)", short_kernel(e["name"])
        else:
            label, site, _ = CALLS[idx]
            key = f"{label} @ {site}"
        r = rows.setdefault(key, dict(site=key, kernels=collections.Counter(), calls=set(), launches=0, ms=0.0, bytes=0))
        r["kernels"][short_kernel(e["name"])] += e.get("dur", 0.0)
        r["launches"] += 1
        r["ms"] += e.get("dur", 0.0) / 1e3
        if idx is not None and idx not in r["calls"]:
            r["calls"].add(idx)
            r["bytes"] += CALLS[idx][2]
    return rows, gpu


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="products", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for trace.json and table.json (default: a new temporary directory)")
    ap.add_argument("--peak", type=float, default=3350.0, help="HBM GB/s (default: H100 SXM data sheet)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("profile_step.py needs a CUDA device")
    if args.out is None:
        args.out = tempfile.mkdtemp(prefix="profile_step_")
    os.makedirs(args.out, exist_ok=True)
    from sgformer_b200 import large as L
    from sgformer_b200.loss import nll_loss_from_logits
    from sgformer_b200.synth import make_graph

    w = bench.WORKLOADS[args.workload]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    # as bench.run_full_batch(parallel='single')
    torch.manual_seed(1234)
    n, d, c, h = w["n"], w["d"], w["c"], w["h"]
    ei = make_graph(n, w["e"], seed=100, device=dev)
    g = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(n, d, generator=g, device=dev)
    y = torch.randint(0, c, (n,), generator=g, device=dev)
    model = L.SGFormer(d, h, c, **bench.model_kwargs(w)).to(dev).set_precision(w["precision"])
    opt = bench._optimizer(model)
    model.train()

    def step():
        opt.zero_grad(set_to_none=True)
        out = model(x, ei)
        loss = nll_loss_from_logits(out, y, None, float(n))
        loss.backward()
        opt.step()
        return loss

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    wrap_kernels()
    step()                      # the wrappers' first calls (and the graph cache) outside the profiled step
    torch.cuda.synchronize()
    CALLS.clear()
    l0 = K.launch_count()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        wall_ms = (time.perf_counter() - t0) * 1e3
    launches = K.launch_count() - l0
    trace = os.path.join(args.out, "trace.json")
    prof.export_chrome_trace(trace)
    rows, gpu = attribute(trace)

    busy = sum(e.get("dur", 0.0) for e in gpu) / 1e3
    gaps = 0.0
    for a, b in zip(gpu, gpu[1:]):
        gaps += max(0.0, b["ts"] - (a["ts"] + a.get("dur", 0.0))) / 1e3
    span = (gpu[-1]["ts"] + gpu[-1].get("dur", 0.0) - gpu[0]["ts"]) / 1e3 if gpu else 0.0
    info = bench.gpu_info(0)
    n_kernels = sum(1 for e in gpu if e["cat"] == "kernel")
    table = []
    for r in sorted(rows.values(), key=lambda r: -r["ms"]):
        gbs = r["bytes"] / (r["ms"] * 1e6) if r["ms"] > 0 and r["bytes"] else 0.0
        table.append(dict(site=r["site"], kernel=r["kernels"].most_common(1)[0][0], calls=len(r["calls"]),
                          launches=r["launches"], ms=r["ms"], gbytes=r["bytes"] / 1e9, gbs=gbs, frac_peak=gbs / args.peak))
    print(f"# {info['name']}, power limit {info['power_limit_w']} W; workload {args.workload}; one eager step "
          f"under the profiler")
    print(f"# wall {wall_ms:.1f} ms (profiled), GPU span {span:.1f} ms, GPU busy {busy:.1f} ms, gaps {gaps:.2f} ms; "
          f"{n_kernels} kernels in the trace ({launches} through the sgformer_b200 C-ABI)")
    hdr = f"{'ms':>8} {'share':>6} {'n':>3} {'GB':>7} {'TB/s':>6} {'peak':>5}  site  [kernel]"
    print(hdr)
    tot_ms = sum(t["ms"] for t in table)
    for t in table:
        frac = f"{t['frac_peak']:5.2f}" if t["gbytes"] else "    -"
        print(f"{t['ms']:8.3f} {t['ms'] / tot_ms:6.1%} {t['launches']:3d} {t['gbytes']:7.2f} {t['gbs'] / 1e3:6.2f} {frac}  "
              f"{t['site']}  [{t['kernel']}]")
    with open(os.path.join(args.out, "table.json"), "w") as fh:
        json.dump(dict(gpu=info, workload=args.workload, wall_ms=wall_ms, span_ms=span, busy_ms=busy, gaps_ms=gaps,
                       kernels=n_kernels, abi_launches=launches, peak_gbs=args.peak, rows=table), fh, indent=1)
    print(f"# trace and table in {args.out}")


if __name__ == "__main__":
    main()
