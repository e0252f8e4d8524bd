"""CPU checks of the GAT backbone: the backward formulas sgf_gat_bwd implements (two passes, no [nnz] arrays) against fp64
autograd of the oracle conv, the parameter naming of the native modules (PyG 2.0-2.3 names, the 1.7.2 / >= 2.4 layouts accepted
by load_state_dict) and the clear errors for what is out of scope."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import gat_oracle as G


def _graph(n, e, seed):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n - 2, (e,), generator=g)
    dst = torch.randint(0, n - 2, (e,), generator=g)
    return torch.stack([torch.cat([src, src[:7], torch.arange(3)]), torch.cat([dst, dst[:7], torch.arange(3)])])


def _kernel_backward(xp, att_s, att_d, ei, g, factor, mean):
    """The arithmetic of sgf_gat_bwd restated per edge in fp64: pass 1 over the in-edges of each target, pass 2 over the
    out-edges of each source, softmax weights rebuilt from the saved log-sum-exp."""
    n, H, C = xp.shape
    a_s, a_d = (xp * att_s).sum(-1), (xp * att_d).sum(-1)
    src, dst = G.gat_edges(ei, n)
    pre = a_s[src] + a_d[dst]
    e = F.leaky_relu(pre, 0.2)
    lse = torch.full((n, H), -float("inf"), dtype=xp.dtype).scatter_reduce(0, dst[:, None].expand_as(e), e, "amax")
    lse = lse + torch.zeros((n, H), dtype=xp.dtype).index_add(0, dst, (e - lse[dst]).exp()).log()
    alpha = (e - lse[dst]).exp()
    lg = torch.where(pre > 0, 1.0, 0.2).to(xp.dtype)
    gh = (g / H).unsqueeze(1).expand(n, H, C) if mean else g.view(n, H, C)
    dalpha = factor * (gh[dst] * xp[src]).sum(-1)
    # pass 1: r_i = sum alpha dalpha, da_dst = sum alpha dalpha lrelu' - r sum alpha lrelu'
    r = torch.zeros((n, H), dtype=xp.dtype).index_add(0, dst, alpha * dalpha)
    da_dst = torch.zeros((n, H), dtype=xp.dtype).index_add(0, dst, alpha * dalpha * lg) - \
        r * torch.zeros((n, H), dtype=xp.dtype).index_add(0, dst, alpha * lg)
    # pass 2: dxp_j = sum alpha d g_i + da_src_j att_src + da_dst_j att_dst, da_src_j = sum alpha (dalpha - r_i) lrelu'
    de = alpha * (dalpha - r[dst])
    da_src = torch.zeros((n, H), dtype=xp.dtype).index_add(0, src, de * lg)
    dxp = torch.zeros_like(xp).index_add(0, src, (alpha * factor)[..., None] * gh[dst])
    dxp = dxp + da_src[..., None] * att_s + da_dst[..., None] * att_d
    return dxp, da_src, da_dst


@pytest.mark.parametrize("heads,concat,p", [(1, True, 0.0), (2, False, 0.0), (8, True, 0.5), (2, False, 0.3)])
def test_backward_formulas_match_autograd(heads, concat, p):
    torch.manual_seed(0)
    n, d, c = 40, 6, 4
    ei = _graph(n, 150, 1)
    conv = G.GATConv(d, c, heads=heads, concat=concat).double()
    x = torch.randn(n, d, dtype=torch.float64)
    xp = (x @ conv.lin_src.weight.detach().t()).view(n, heads, c).requires_grad_(True)
    ne = G.gat_edges(ei, n).shape[1]
    factor = (torch.rand(ne, heads, dtype=torch.float64) >= p).double() / (1 - p)
    att_s = conv.att_src.detach().clone().requires_grad_(True)
    att_d = conv.att_dst.detach().clone().requires_grad_(True)

    def f(xp_, as_, ad_):
        # the conv after its projection, so that xp, att_src and att_dst are the differentiated leaves
        a_s, a_d = (xp_ * as_).sum(-1), (xp_ * ad_).sum(-1)
        src, dst = G.gat_edges(ei, n)
        e = F.leaky_relu(a_s[src] + a_d[dst], 0.2)
        m = torch.full((n, heads), -float("inf"), dtype=e.dtype).scatter_reduce(0, dst[:, None].expand_as(e), e, "amax")
        ex = (e - m[dst]).exp()
        alpha = ex / torch.zeros((n, heads), dtype=e.dtype).index_add(0, dst, ex)[dst] * factor
        out = torch.zeros_like(xp_).index_add(0, dst, alpha[..., None] * xp_[src])
        return out.reshape(n, heads * c) if concat else out.mean(1)

    out = f(xp, att_s, att_d)
    g = torch.randn_like(out)
    out.backward(g)
    dxp, da_src, da_dst = _kernel_backward(xp.detach(), att_s.detach(), att_d.detach(), ei, g, factor, not concat)
    assert torch.allclose(dxp, xp.grad, rtol=1e-7, atol=1e-7), (dxp - xp.grad).abs().max()
    xpd = xp.detach()
    assert torch.allclose((da_src[..., None] * xpd).sum(0), att_s.grad[0], rtol=1e-7, atol=1e-7)
    assert torch.allclose((da_dst[..., None] * xpd).sum(0), att_d.grad[0], rtol=1e-7, atol=1e-7)


def test_oracle_gat_edges():
    ei = torch.tensor([[0, 1, 1, 2, 2], [1, 1, 0, 2, 0]])
    assert G.gat_edges(ei, 4).tolist() == [[0, 1, 2, 0, 1, 2, 3], [1, 0, 0, 0, 1, 2, 3]]


def test_native_gat_names_and_layouts():
    from sgformer_b200 import medium as M
    ours = M.GAT(10, 8, 8, num_layers=3, heads=2, out_heads=2, use_bn=True)
    ref = G.GAT(10, 8, 8, num_layers=3, heads=2, out_heads=2, use_bn=True)
    assert list(ours.state_dict().keys()) == list(ref.state_dict().keys())
    for k, v in ref.state_dict().items():
        assert ours.state_dict()[k].shape == v.shape, k
    sd = ref.state_dict()
    ours.load_state_dict(sd)
    assert all(torch.equal(a, b) for a, b in zip(ours.state_dict().values(), sd.values()))
    # PyG 1.7.2: lin_l / lin_r / att_l / att_r;  PyG >= 2.4: lin
    old = {}
    for k, v in sd.items():
        if "lin_dst" in k:
            continue
        k = k.replace("lin_src.weight", "lin_l.weight").replace("att_src", "att_l").replace("att_dst", "att_r")
        old[k] = v + 1.0 if v.is_floating_point() else v
    ours.load_state_dict(old)
    assert torch.equal(ours.convs[1].lin_src.weight, sd["convs.1.lin_src.weight"] + 1.0)
    assert torch.equal(ours.convs[2].att_dst, sd["convs.2.att_dst"] + 1.0)
    new = {k.replace("lin_src.weight", "lin.weight"): v for k, v in sd.items() if "lin_dst" not in k}
    ours.load_state_dict(new)
    assert torch.equal(ours.convs[0].lin_dst.weight, sd["convs.0.lin_src.weight"])
    cp = copy.deepcopy(ours)
    assert cp.convs[0].lin_src is cp.convs[0].lin_dst and cp.convs[0].lin_src is not ours.convs[0].lin_src
    ours.reset_parameters()
    assert torch.count_nonzero(ours.convs[0].bias) == 0


def test_out_of_scope_raises():
    from sgformer_b200 import medium as M
    with pytest.raises(NotImplementedError, match="edge_attr"):
        M.GATConv(4, 4, edge_dim=3)
    with pytest.raises(NotImplementedError, match="tuple"):
        M.GATConv((4, 5), 4)
    with pytest.raises(NotImplementedError, match="return_attention_weights"):
        M.GATConv(4, 4)(torch.zeros(2, 4), torch.zeros(2, 0, dtype=torch.long), return_attention_weights=True)


def test_gat_config_kind():
    from sgformer_b200.config import make_config
    assert make_config("medium", 4, 8, 3)["gnn_kind"] == "gcn"
    with pytest.raises(ValueError):
        make_config("medium", 4, 8, 3, gnn_kind="gin")
