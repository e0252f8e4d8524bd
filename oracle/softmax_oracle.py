"""Plain-torch restatement of SGFormerSOFT's attention branch (medium/ablation/oursSOFT.py:14-165) for the tests: any dtype
(fp64 for the references), functional over a state_dict, dropout off.  As in the reference, the softmax runs over the last axis
of the [N, L, H] scores: over the heads (tests/test_softmax_ablation.py checks this against tests/golden/sgformer_softmax.pt,
made from the unmodified oursSOFT.py)."""
import torch
import torch.nn.functional as F


def softmax_attention(qs, ks, vs):
    """oursSOFT.py:14-34 (qs, ks [N, H, M], vs [N, H, D] or [N, 1, D]) -> ([N, H, D], [N, N] head mean of the weights)."""
    qs = qs / torch.norm(qs, p=2)
    ks = ks / torch.norm(ks, p=2)
    w = F.softmax(torch.einsum("nhm,lhm->nlh", qs, ks), dim=-1)
    return torch.einsum("nlh,lhd->nhd", w, vs.expand(-1, qs.shape[1], -1)), w.mean(dim=-1)


def trans_conv(sd, x, num_layers, num_heads, alpha=0.5, use_bn=True, use_residual=True, use_weight=True, prefix="trans_conv.",
               attentions=None):
    """TransConv.forward (oursSOFT.py:121-148) at dropout 0; `attentions` (a list) collects each layer's [N, N] weights."""
    h = sd[prefix + "fcs.0.weight"].shape[0]
    x = F.linear(x, sd[prefix + "fcs.0.weight"], sd[prefix + "fcs.0.bias"])
    if use_bn:
        x = F.layer_norm(x, (h,), sd[prefix + "bns.0.weight"], sd[prefix + "bns.0.bias"])
    x = F.relu(x)
    prev = x
    for i in range(num_layers):
        lp = f"{prefix}convs.{i}."
        q = F.linear(x, sd[lp + "Wq.weight"], sd[lp + "Wq.bias"]).reshape(-1, num_heads, h)
        k = F.linear(x, sd[lp + "Wk.weight"], sd[lp + "Wk.bias"]).reshape(-1, num_heads, h)
        v = F.linear(x, sd[lp + "Wv.weight"], sd[lp + "Wv.bias"]).reshape(-1, num_heads, h) if use_weight else x.reshape(-1, 1, h)
        o, att = softmax_attention(q, k, v)
        if attentions is not None:
            attentions.append(att)
        x = o.mean(dim=1)
        if use_residual:
            x = alpha * x + (1 - alpha) * prev
        if use_bn:
            x = F.layer_norm(x, (h,), sd[f"{prefix}bns.{i + 1}.weight"], sd[f"{prefix}bns.{i + 1}.bias"])
        prev = x
    return x


def sgformer_soft(sd, x, num_layers, num_heads, **kw):
    """SGFormerSOFT.forward with use_graph=False (oursSOFT.py:190-201)."""
    return F.linear(trans_conv(sd, x, num_layers, num_heads, **kw), sd["fc.weight"], sd["fc.bias"])
