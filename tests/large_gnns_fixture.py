"""Loader of tests/golden/large_gnns.pt (tests/make_golden_large_gnns.py), the fp64 oracle run of one case, and the kernel
emulation with the unscaled SpMM, shared by tests/test_large_gnns.py (CPU) and tests/test_gpu_large_gnns.py."""
import os
import types

import torch

import kernel_emu
from oracle import large_gnns_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _unflat(d):
    out, o = {}, 0
    for name, shape in zip(d["names"], d["shapes"]):
        k = 1
        for s in shape:
            k *= s
        out[name] = d["flat"][o:o + k].reshape(shape).clone()
        o += k
    return out


def load():
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "large_gnns.pt"), weights_only=False)
    for name, c in fx.items():
        if name == "__trees__":
            continue
        c["state_dict"] = _unflat(c["state_dict"])
        c["grads"] = _unflat(c["grads"])
        c["buffers_after_train"] = _unflat(c["buffers_after_train"]) if c["buffers_after_train"] else {}
        c["edge_index"] = c["edge_index"].long()
    return fx


def state_dict_as_loaded(c):
    """The fixture's state_dict with num_batches_tracked back to int64 (the flat storage holds fp32)."""
    return {k: (v.long() if k.endswith("num_batches_tracked") else v) for k, v in c["state_dict"].items()}


def oracle_run(c, dtype, training):
    """-> (logits, {param: grad}, grad_x, buffers) of the oracle in `dtype`; grads only when training."""
    sd = {k: (v.to(dtype).clone().requires_grad_(training and "running" not in k and "num_batches" not in k)
              if v.is_floating_point() else v) for k, v in c["state_dict"].items()}
    x = c["x"].to(dtype).clone().requires_grad_(training)
    stats = {}
    g = c["gcn"]
    out = O.gcn_large(x, c["edge_index"], sd, g["num_layers"], g["use_bn"], g["save_mem"], training, stats_out=stats)
    if not training:
        return out.detach(), {}, None, {}
    (out * c["loss_weight"].to(dtype)).sum().backward()
    grads = {k: v.grad for k, v in sd.items() if isinstance(v, torch.Tensor) and v.grad is not None}
    return out.detach(), grads, x.grad, stats


def emulated_kernels():
    """kernel_emu plus the unscaled SpMM (sgf_spmm_sum: the plain sum over the CSR as built)."""
    m = types.ModuleType("kernel_emu_large_gnns")
    m.__dict__.update(kernel_emu.__dict__)
    m.spmm_sum = lambda rowptr, col, x, out=None, heavy=None: kernel_emu.spmm(rowptr, col, None, x, out)
    return m
