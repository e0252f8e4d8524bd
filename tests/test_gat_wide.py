"""CPU checks of GAT layers wider than one launch of the GAT kernels (engine.gat_groups): the head-group plan, and the grouped and
zero-padded schedule (engine.gat_forward / gat_backward inside GraphBranchFn and SGFormerFn) with the kernels replaced by their
torch-CPU contracts (tests/kernel_emu_gat.py) against oracle/gat_oracle.py in fp64.

The bf16 cases run the bf16 plan (heads padded to 8 channels, groups of up to 1024 channels) in the emulator's fp32 arithmetic, so
that they can be held to the same 1e-5; bf16 rounding is checked on the device (tests/test_gpu_gat_wide.py)."""
import math
import types

import pytest
import torch
import torch.nn.functional as F

import gat_widths as W
import kernel_emu_gat as emu
from oracle import gat_oracle as G
from oracle import sgformer_oracle as O
from sgformer_b200 import engine as E
from sgformer_b200 import functional as Fn
from sgformer_b200 import medium as M
from sgformer_b200.dist import SINGLE


# ------------------------------------------------------------------------------------------------
# the group plan
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_group_plan_covers_every_head_within_the_launch_limits(dtype):
    vn, row_max = (8, 1024) if dtype == "bf16" else (4, 512)
    for heads in list(range(1, 21)) + [24, 31, 32, 64]:
        for c in sorted(set(range(1, 70)) | {100, 128, 250, 256, 300, 511, 512, 513, 1000, 1024}):
            cp_want = -(-c // vn) * vn
            if cp_want > row_max:
                with pytest.raises(ValueError, match="one head must fit one launch"):
                    E.gat_groups(dtype, heads, c)
                continue
            cp, groups = E.gat_groups(dtype, heads, c)
            assert cp == cp_want
            assert [h for h0, hg in groups for h in range(h0, h0 + hg)] == list(range(heads)), (heads, c, groups)
            assert all(W.geometry(dtype, hg, cp) is not None for _, hg in groups), (heads, c, groups)
            sizes = [hg for _, hg in groups]
            assert max(sizes) - min(sizes) <= 1 and sizes == sorted(sizes, reverse=True)
            per = min(W.max_heads(), row_max // cp)
            assert len(groups) == -(-heads // per), "as few groups as the limits allow"
            if W.geometry(dtype, heads, c) is not None:         # fits one launch today: one group, unpadded
                assert groups == [(0, heads)] and cp == c
            if c % vn == 0 and heads <= W.max_heads() and heads * c <= row_max:
                assert groups == [(0, heads)]


def test_group_plan_of_the_issue_widths():
    assert E.gat_groups("fp32", 4, 256) == (256, [(0, 2), (2, 2)])
    assert E.gat_groups("fp32", 8, 128) == (128, [(0, 4), (4, 4)])
    assert E.gat_groups("fp32", 16, 64) == (64, [(0, 8), (8, 8)])
    assert E.gat_groups("fp32", 3, 250) == (252, [(0, 2), (2, 1)])
    assert E.gat_groups("bf16", 8, 256) == (256, [(0, 4), (4, 4)])
    assert E.gat_groups("bf16", 3, 100) == (104, [(0, 3)])
    assert E.gat_groups("fp32", 10, 7) == (8, [(0, 5), (5, 5)])
    assert E.gat_groups("fp32", 8, 64) == (64, [(0, 8)])
    with pytest.raises(ValueError, match="set_precision\\('bf16'\\)"):
        E.gat_groups("fp32", 1, 1024)


def test_single_head_wider_than_a_launch_is_refused_by_name():
    P = {"l.lin_src.weight": torch.zeros(1024, 16), "l.att_src": torch.zeros(1, 1, 1024), "l.att_dst": torch.zeros(1, 1, 1024),
         "l.bias": torch.zeros(1024)}
    with pytest.raises(ValueError, match="GAT layer 0: .*out_channels at most 512"):
        E._gat_layer(P, "l.", 1, 1024, False, E.FP32, 0)
    assert E._gat_layer(P, "l.", 1, 1024, False, E.BF16, 0)[0] == 1024


def test_padding_round_trips():
    t = torch.randn(3 * 5, 7)
    p = E._pad_heads(t, 3, 5, 8)
    assert p.shape == (24, 7) and torch.equal(p.view(3, 8, 7)[:, 5:], torch.zeros(3, 3, 7))
    assert torch.equal(E._unpad_heads(p, 3, 5, 8), t)
    q = E._pad_heads(t.t(), 3, 5, 8, dim=1, fill=1.0)
    assert q.shape == (7, 24) and torch.equal(q.view(7, 3, 8)[:, :, 5:], torch.ones(7, 3, 3))
    assert torch.equal(E._unpad_heads(q, 3, 5, 8, dim=1), t.t())
    assert E._pad_heads(t, 3, 5, 5) is t


# ------------------------------------------------------------------------------------------------
# the schedule on the emulated kernels
# ------------------------------------------------------------------------------------------------
def _placed(fn, key, index=0):
    """An emulated launcher with the output-placement keyword of kernels.py: the result is written into the given view."""
    def f(*a, **kw):
        dst = kw.pop(key, None)
        r = fn(*a, **kw)
        if dst is None:
            return r
        r = list(r)
        dst.copy_(r[index])
        r[index] = dst
        return tuple(r)
    return f


K_WIDE = types.SimpleNamespace(**{k: v for k, v in vars(emu).items() if not k.startswith("__")})
K_WIDE.gat_fwd = _placed(emu.gat_fwd, "out")
K_WIDE.gat_bwd = _placed(emu.gat_bwd, "dxp_out")
K_WIDE.bn_fwd = _placed(emu.bn_fwd, "y_out")
K_WIDE.bn_bwd = _placed(emu.bn_bwd, "dz_out")


class _Fp32Arith(E.Precision):
    """A precision's plan (group sizes, padding) run with fp32 activations, as the emulator computes."""
    @property
    def act_dtype(self):
        return torch.float32

    @property
    def planes(self):
        return 3


PREC = {"fp32": E.FP32, "bf16": _Fp32Arith("bf16")}


class Data:
    def __init__(self, x, ei):
        self.graph = {"node_feat": x, "edge_index": ei, "num_nodes": x.shape[0]}


def _graph(n=37, e=160, seed=3):
    """Directed: duplicate edges, existing self loops, an isolated node."""
    g = torch.Generator().manual_seed(seed)
    src, dst = torch.randint(0, n - 1, (e,), generator=g), torch.randint(0, n - 1, (e,), generator=g)
    return torch.stack([torch.cat([src, src[:9], torch.arange(4)]), torch.cat([dst, dst[:9], torch.arange(4)])])


def _ref_gat(d, h, c, layers, heads, out_heads, use_bn, seed):
    torch.manual_seed(seed)
    ref = G.GAT(d, h, c, num_layers=layers, dropout=0.0, use_bn=use_bn, heads=heads, out_heads=out_heads).double()
    with torch.no_grad():
        for conv in ref.convs:
            conv.bias.normal_(0, 0.1)
        for bn in ref.bns:
            bn.weight.uniform_(0.5, 1.5); bn.bias.normal_(0, 0.1)
            bn.running_mean.normal_(0, 0.1); bn.running_var.uniform_(0.5, 1.5)
    return ref


def _ours_gat(ref, d, h, c, layers, heads, out_heads, use_bn):
    ours = M.GAT(d, h, c, num_layers=layers, dropout=0.0, use_bn=use_bn, heads=heads, out_heads=out_heads)
    ours.load_state_dict({k: v.float() if v.is_floating_point() else v for k, v in ref.state_dict().items()})
    return ours


def _close(a, b, what, floor=1e-3, rtol=1e-5):
    a, b = a.detach().double(), b.detach().double()
    assert a.shape == b.shape, f"{what}: shape {tuple(a.shape)} vs {tuple(b.shape)}"
    err = (a - b).abs().max().item()
    assert err <= rtol * max(b.abs().max().item(), floor), f"{what}: max err {err:.3e} of {b.abs().max().item():.3e}"


def _run_gat(model, x, ei, prec, training):
    names, tensors = M._gat_flat(model, "gnn.")
    cfg = M.make_config("medium", x.shape[1], model.convs[0].lin_src.weight.shape[0], model.convs[-1].out_channels,
                        **model._cfg_kw())
    return Fn.GraphBranchFn.apply(x, emu.EmuGraph(ei, x.shape[0], 1), cfg, prec, training, "gat", "gnn.", names, *tensors)


def _step(run, model, x, lw):
    """eval logits, train logits, parameter gradients, input gradient and running buffers after the train step."""
    model.eval()
    with torch.no_grad():
        out_eval = run(x, False)
    model.train()
    xg = x.clone().requires_grad_(True)
    out = run(xg, True)
    (out * lw).sum().backward()
    grads = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    grads["__x__"] = xg.grad
    buffers = {k: v.clone() for k, v in model.state_dict().items() if "running" in k}
    return dict(out_eval=out_eval.detach(), out_train=out.detach(), grads=grads, buffers=buffers)


def _compare(got, ref, what):
    _close(got["out_eval"], ref["out_eval"], f"eval logits [{what}]")
    _close(got["out_train"], ref["out_train"], f"train logits [{what}]")
    gmax = max(g.abs().max().item() for g in ref["grads"].values())
    assert set(got["grads"]) == set(ref["grads"]), sorted(set(got["grads"]) ^ set(ref["grads"]))
    for k, g in ref["grads"].items():
        _close(got["grads"][k], g, f"{k} [{what}]", floor=gmax)
    assert set(got["buffers"]) == set(ref["buffers"])
    for k, v in ref["buffers"].items():
        _close(got["buffers"][k], v, f"{k} [{what}]", floor=1.0)


# (precision, heads, hidden): the widths of the issue's table; none fits one launch
WIDE = [("fp32", 4, 256), ("fp32", 8, 128), ("fp32", 16, 64), ("fp32", 3, 250), ("bf16", 8, 256), ("bf16", 16, 64), ("bf16", 3, 100)]
# (out_heads, out_channels) of the last, head-mean conv: two groups of 5 heads, and two heads of 7 zero-padded classes
HEADS = [(10, 6), (2, 7)]
CASES = [(w, L, bn, hd) for w in WIDE for L in (2, 3) for bn in (True, False) for hd in HEADS]


def test_wide_cases_need_the_group_schedule():
    for dt, h, c in WIDE:
        cp, groups = E.gat_groups(dt, h, c)
        assert len(groups) > 1 or cp != c, (dt, h, c)
    assert len(E.gat_groups("fp32", 10, 6)[1]) == 2 and E.gat_groups("fp32", 2, 7)[0] == 8


@pytest.mark.parametrize("wide,layers,use_bn,head", CASES,
                         ids=[f"{w[0]}-{w[1]}x{w[2]}-L{L}-bn{int(bn)}-oh{hd[0]}c{hd[1]}" for w, L, bn, hd in CASES])
def test_emulated_wide_gat_matches_the_oracle(monkeypatch, wide, layers, use_bn, head):
    monkeypatch.setattr(E, "K", K_WIDE)
    monkeypatch.setattr(Fn, "K", K_WIDE)
    dt, heads, h = wide
    out_heads, c = head
    n, d = 37, 12
    ei = _graph()
    seed = heads * 1000 + h + layers
    ref = _ref_gat(d, h, c, layers, heads, out_heads, use_bn, seed)
    ours = _ours_gat(ref, d, h, c, layers, heads, out_heads, use_bn)
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(n, d, generator=gen, dtype=torch.float64)
    lw = torch.randn(n, c, generator=gen, dtype=torch.float64)
    r = _step(lambda xx, tr: ref(Data(xx, ei)), ref, x, lw)
    got = _step(lambda xx, tr: _run_gat(ours, xx, ei, PREC[dt], tr), ours, x.float(), lw.float())
    _compare(got, r, f"{wide} L{layers} bn={use_bn} head={head}")
    # the module keeps the reference's unpadded shapes
    assert all(ours.state_dict()[k].shape == v.shape for k, v in ref.state_dict().items())


# SGFormer's own layers keep their width rule (engine.check_width): hidden a multiple of 4 / 8, at most 512 / 1024
SG_CASES = [(w, agg, oh) for w in [("fp32", 4, 256), ("fp32", 8, 128), ("fp32", 16, 64), ("bf16", 8, 256)] for agg in ("add", "cat")
            for oh in (1, 4)]


@pytest.mark.parametrize("wide,aggregate,out_heads", SG_CASES,
                         ids=[f"{w[0]}-{w[1]}x{w[2]}-{a}-oh{oh}" for w, a, oh in SG_CASES])
def test_emulated_wide_sgformer_gat_matches_the_oracle(monkeypatch, wide, aggregate, out_heads):
    """SGFormer(gnn=GAT): the GAT branch's last conv is a head mean over `hidden` channels (out_heads of them: a wide head mean
    over 2 KB rows at 4 x 256 fp32 and 4 x 128 fp32)."""
    monkeypatch.setattr(E, "K", K_WIDE)
    monkeypatch.setattr(Fn, "K", K_WIDE)
    dt, heads, h = wide
    n, d, c = 37, 12, 5
    ei = _graph(seed=9)
    ref_gnn = _ref_gat(d, h, h, 2, heads, out_heads, True, 11)
    gnn = _ours_gat(ref_gnn, d, h, h, 2, heads, out_heads, True)
    model = M.SGFormer(d, h, c, num_layers=1, num_heads=1, alpha=0.3, dropout=0.0, use_bn=True, gnn=gnn, aggregate=aggregate,
                       graph_weight=0.7)
    cfg = O.make_config("medium", d, h, c, num_layers=1, num_heads=1, alpha=0.3, dropout=0.0, use_bn=True, aggregate=aggregate,
                        graph_weight=0.7)
    sd = {k: v.detach().double().clone() for k, v in model.state_dict().items() if not k.startswith("gnn.")}

    class Ref(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.gnn = ref_gnn
            self.p = torch.nn.ParameterDict({k.replace(".", "__"): torch.nn.Parameter(v) for k, v in sd.items()})

        def forward(self, data):
            x, ei_ = data.graph["node_feat"], data.graph["edge_index"]
            P = {k.replace("__", "."): v for k, v in self.p.items()}
            x1 = O.trans_conv(x, P, cfg, self.training)
            x2 = self.gnn(data)
            hcat = 0.7 * x2 + 0.3 * x1 if aggregate == "add" else torch.cat([x1, x2], 1)
            return F.linear(hcat, P["fc.weight"], P["fc.bias"])
    ref = Ref()

    def run(xx, training):
        tn, tt = model.trans_conv._flat("trans_conv.")
        gn, gt = M._gat_flat(model.gnn, "gnn.")
        mcfg = model._cfg(len(model.gnn.convs), float(model.gnn.dropout), bool(model.gnn.use_bn), "gat")
        names = tuple(tn) + tuple("fc." + k for k in model.fc._parameters) + tuple(gn)
        tensors = list(tt) + list(model.fc._parameters.values()) + list(gt)
        return Fn.SGFormerFn.apply(xx, emu.EmuGraph(ei, xx.shape[0], 1), mcfg, PREC[dt], training, SINGLE, names, *tensors)

    gen = torch.Generator().manual_seed(5)
    x = torch.randn(n, d, generator=gen, dtype=torch.float64)
    lw = torch.randn(n, c, generator=gen, dtype=torch.float64) / math.sqrt(n)
    r = _step(lambda xx, tr: ref(Data(xx, ei)), ref, x, lw)
    r["grads"] = {(k[2:].replace("__", ".") if k.startswith("p.") else k): v for k, v in r["grads"].items()}
    got = _step(run, model, x.float(), lw.float())
    _compare(got, r, f"SGFormer {wide} {aggregate} out_heads={out_heads}")
