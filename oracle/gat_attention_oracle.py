"""Plain-torch restatement of SGFormerGAT's attention branch (medium/ablation/oursGAT.py:13-183) for the tests: any dtype (fp64
for the references), functional over a state_dict, dropout off.  As in the reference, the softmax runs over the last axis of the
[N, L, H] scores: over the heads (tests/test_gat_attention_ablation.py checks this against tests/golden/sgformer_gat_attention.pt,
made from the unmodified oursGAT.py).  The layers' own Wq / Wk / Wv never reach the output and are not read."""
import torch
import torch.nn.functional as F


def gat_attention(qs, ks, vs):
    """GATAttention's core (oursGAT.py:36-43): qs, ks [N, H, dk], vs [N, H, D] -> [N, H, D].  The scale is the reference's:
    the square root of an fp32 tensor holding dk."""
    dk = qs.shape[2]
    scores = torch.einsum("nhm,lhm->nlh", qs, ks) / torch.sqrt(torch.tensor([float(dk)], dtype=torch.float32)).to(qs.device)
    return torch.einsum("nlh,lhd->nhd", F.softmax(scores, dim=-1), vs)


def layer(sd, lp, x, num_heads, use_weight=True):
    """TransConvLayer.forward (oursGAT.py:85-107) of the layer with state_dict prefix lp -> [N, h]."""
    a = lp + "attention.attention."
    h = x.shape[1]
    dk = h // num_heads
    u = F.linear(x, sd[lp + "attention.Wv.weight"], sd[lp + "attention.Wv.bias"]) if use_weight else x
    q = F.linear(x, sd[a + "Wq.weight"], sd[a + "Wq.bias"]).view(-1, num_heads, dk)
    k = F.linear(x, sd[a + "Wk.weight"], sd[a + "Wk.bias"]).view(-1, num_heads, dk)
    v = F.linear(u, sd[a + "Wv.weight"], sd[a + "Wv.bias"]).view(-1, num_heads, sd[a + "Wv.weight"].shape[0] // num_heads)
    return gat_attention(q, k, v).mean(dim=1)


def trans_conv(sd, x, num_layers, num_heads, alpha=0.5, use_bn=True, use_residual=True, use_weight=True, prefix="trans_conv."):
    """TransConv.forward (oursGAT.py:139-166) at dropout 0."""
    h = sd[prefix + "fcs.0.weight"].shape[0]
    x = F.linear(x, sd[prefix + "fcs.0.weight"], sd[prefix + "fcs.0.bias"])
    if use_bn:
        x = F.layer_norm(x, (h,), sd[prefix + "bns.0.weight"], sd[prefix + "bns.0.bias"])
    x = F.relu(x)
    prev = x
    for i in range(num_layers):
        x = layer(sd, f"{prefix}convs.{i}.", x, num_heads, use_weight)
        if use_residual:
            x = alpha * x + (1 - alpha) * prev
        if use_bn:
            x = F.layer_norm(x, (h,), sd[f"{prefix}bns.{i + 1}.weight"], sd[f"{prefix}bns.{i + 1}.bias"])
        prev = x
    return x


def sgformer_gat(sd, x, num_layers, num_heads, **kw):
    """SGFormerGAT.forward with use_graph=False (oursGAT.py:208-219)."""
    return F.linear(trans_conv(sd, x, num_layers, num_heads, **kw), sd["fc.weight"], sd["fc.bias"])
