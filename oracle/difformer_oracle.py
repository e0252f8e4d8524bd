"""Plain-torch restatement of DIFFormer with the `simple` kernel and one head (medium/difformer.py), written from its
mathematics: the checker the kernel path is compared with, and the torch baseline of scripts/bench_difformer.py.

Layer i with input x (= the previous layer's output, x0 = the input MLP's output):
    q, k, v = Linear(x)  (v = x when use_weight is off)
    attn    = (q~ (k~^T v) + 1 (sum_l v_l)) / (q~ . sum_l k~_l + N),  q~ = q / ||q||_F, k~ = k / ||k||_F
    y       = D^-1/2 A D^-1/2 v  over the edges (src -> dst), D = in-degree at dst, no self loops, 1/sqrt(0) -> 0
    c       = attn + y  (graph_weight <= 0) | (1-gw) attn + gw y  (graph_weight > 0) | attn  (use_graph off)
    c      += x0 if use_source;   x' = alpha c + (1-alpha) x if use_residual;   x' = LayerNorm(x') if use_bn;   dropout
Input: x0 = dropout(relu(LayerNorm?(fcs.0 x))); output: fcs.1 x_L."""
import torch
import torch.nn.functional as F

DEFAULTS = dict(num_layers=2, alpha=0.5, dropout=0.5, use_bn=True, use_residual=True, use_weight=True, use_graph=True,
                graph_weight=-1.0, use_source=False)


def make_config(in_channels, hidden, out_channels, **kw):
    cfg = dict(DEFAULTS)
    for k in kw:
        if k not in cfg:
            raise KeyError(k)
    cfg.update(kw)
    cfg.update(in_channels=in_channels, hidden=hidden, out_channels=out_channels)
    return cfg


def gcn_aggregate(v, edge_index, n):
    src, dst = edge_index[0], edge_index[1]
    deg = torch.bincount(dst, minlength=n).to(v.dtype)
    dinv = torch.where(deg > 0, deg.clamp_min(1).rsqrt(), torch.zeros_like(deg))
    w = dinv[dst] * dinv[src]
    return torch.zeros_like(v).index_add_(0, dst, v[src] * w[:, None])


def simple_attention(q, k, v):
    n = q.shape[0]
    qn, kn = q / torch.linalg.vector_norm(q), k / torch.linalg.vector_norm(k)
    num = qn @ (kn.t() @ v) + v.sum(0, keepdim=True)
    den = qn @ kn.sum(0) + n
    return num / den[:, None]


def attention_matrix(q, k):
    n = q.shape[0]
    qn, kn = q / torch.linalg.vector_norm(q), k / torch.linalg.vector_norm(k)
    return (qn @ kn.t()) / (qn @ kn.sum(0) + n)[:, None]


def _lin(sd, name, x):
    return x @ sd[name + ".weight"].t() + sd[name + ".bias"]


def _ln(sd, name, x, cfg):
    return F.layer_norm(x, x.shape[-1:], sd[name + ".weight"], sd[name + ".bias"], 1e-5) if cfg["use_bn"] else x


def _layer(cfg, sd, i, x, x0, edge_index, with_graph=True):
    lp = f"convs.{i}."
    q, k = _lin(sd, lp + "Wq", x), _lin(sd, lp + "Wk", x)
    v = _lin(sd, lp + "Wv", x) if cfg["use_weight"] else x
    att = simple_attention(q, k, v)
    if cfg["use_graph"] and with_graph:
        y = gcn_aggregate(v, edge_index, x.shape[0])
        gw = float(cfg["graph_weight"])
        c = (1 - gw) * att + gw * y if gw > 0 else att + y
    else:
        c = att
    if cfg["use_source"]:
        c = c + x0
    if cfg["use_residual"]:
        c = cfg["alpha"] * c + (1 - cfg["alpha"]) * x
    return _ln(sd, f"bns.{i + 1}", c, cfg), (q, k)


def _dropout(x, p, training):
    return F.dropout(x, p=p, training=training)


def difformer_forward(cfg, sd, x, edge_index, training=False):
    p = cfg["dropout"]
    h = _dropout(F.relu(_ln(sd, "bns.0", _lin(sd, "fcs.0", x), cfg)), p, training)
    x0 = h
    for i in range(cfg["num_layers"]):
        h, _ = _layer(cfg, sd, i, h, x0, edge_index)
        h = _dropout(h, p, training)
    return _lin(sd, "fcs.1", h)


def difformer_attentions(cfg, sd, x):
    """get_attentions for use_graph=False -> [L, N, N, 1]."""
    h = F.relu(_ln(sd, "bns.0", _lin(sd, "fcs.0", x), cfg))
    x0, out = h, []
    for i in range(cfg["num_layers"]):
        h, (q, k) = _layer(cfg, sd, i, h, x0, None, with_graph=False)
        out.append(attention_matrix(q, k))
    return torch.stack(out, 0).unsqueeze(-1)


def init_state_dict(cfg, seed=0):
    """Random parameters with the reference's state_dict keys (LayerNorm affine perturbed away from 1/0)."""
    g = torch.Generator().manual_seed(seed)
    d, h, c = cfg["in_channels"], cfg["hidden"], cfg["out_channels"]

    def lin(o, i):
        b = 1.0 / i ** 0.5
        return (torch.rand(o, i, generator=g) * 2 - 1) * b, (torch.rand(o, generator=g) * 2 - 1) * b

    sd = {}
    sd["fcs.0.weight"], sd["fcs.0.bias"] = lin(h, d)
    for i in range(cfg["num_layers"]):
        for nm in ("Wk", "Wq") + (("Wv",) if cfg["use_weight"] else ()):
            sd[f"convs.{i}.{nm}.weight"], sd[f"convs.{i}.{nm}.bias"] = lin(h, h)
    for i in range(cfg["num_layers"] + 1):
        sd[f"bns.{i}.weight"] = 1 + 0.1 * torch.randn(h, generator=g)
        sd[f"bns.{i}.bias"] = 0.1 * torch.randn(h, generator=g)
    sd["fcs.1.weight"], sd["fcs.1.bias"] = lin(c, h)
    return sd
