"""The attentive probe of dinov3_jax.eval.attentive in float64: `unfolded` is the probe as written (keys and values of
every token, autograd), `folded` restates the fold of csrc/attentive.cu (keys folded into the query, values out of the
sum, the token pass's backward written out as the kernels compute it).  Parameters are a dict of the probe's names
(nn.Linear weights are [out, in])."""
import math

import torch
import torch.nn.functional as F

EPS = 1e-6
NAMES = ("Wq", "Wk", "Wv", "Wo", "W1", "W2", "Wc", "e", "q0", "g1", "b1", "bq", "bv", "bo", "g2", "b2", "bf1", "bf2",
         "bc")


def make_params(D, H, T, C, seed, query_scale=1.0, dtype=torch.float64):
    """Random parameters (LN scales around 1, everything else around 0); `query_scale` scales Wq, so the scores grow
    with it while z = q0 + ... keeps its size."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, std=0.05: torch.randn(*s, generator=g, dtype=dtype) * std
    Fd = 4 * D
    p = {"Wq": r(D, D, std=query_scale / math.sqrt(D)), "Wk": r(D, D, std=1 / math.sqrt(D)),
         "Wv": r(D, D, std=1 / math.sqrt(D)), "Wo": r(D, D, std=1 / math.sqrt(D)), "W1": r(Fd, D, std=1 / math.sqrt(D)), "W2": r(D, Fd, std=1 / math.sqrt(Fd)),
         "Wc": r(C, D, std=1 / math.sqrt(D)), "e": r(T, D, std=0.3), "q0": r(D, std=1.0),
         "g1": 1 + r(D, std=0.2), "b1": r(D, std=0.2), "bq": r(D), "bv": r(D), "bo": r(D), "g2": 1 + r(D, std=0.2),
         "b2": r(D, std=0.2), "bf1": r(Fd), "bf2": r(D), "bc": r(C)}
    return p


def _head(p, z, labels):
    """z [B, D] after the attention -> (logits, mean cross-entropy)."""
    D = z.shape[1]
    h = F.gelu(F.linear(F.layer_norm(z, (D,), p["g2"], p["b2"], EPS), p["W1"], p["bf1"]))
    z2 = z + F.linear(h, p["W2"], p["bf2"])
    logits = F.linear(z2, p["Wc"], p["bc"])
    return logits, F.cross_entropy(logits, labels)


def unfolded(params, x, T, H, labels):
    """{"a": [B, D] pooled output (before Wo), "logits", "loss", "grads": {name: tensor}} with autograd."""
    p = {k: v.detach().clone().double().requires_grad_(True) for k, v in params.items()}
    x = x.double()
    B, N, D = x.shape
    P, dh = N // T, D // H
    u = x + p["e"].repeat_interleave(P, 0)[None]
    y = F.layer_norm(u, (D,), p["g1"], p["b1"], EPS)
    q = F.linear(p["q0"], p["Wq"], p["bq"])
    k = F.linear(y, p["Wk"]).view(B, N, H, dh)
    v = F.linear(y, p["Wv"], p["bv"]).view(B, N, H, dh)
    s = torch.einsum("hd,bnhd->bhn", q.view(H, dh), k) / math.sqrt(dh)
    a = torch.einsum("bhn,bnhd->bhd", s.softmax(-1), v).reshape(B, D)
    z = p["q0"] + F.linear(a, p["Wo"], p["bo"])
    logits, loss = _head(p, z, labels)
    loss.backward()
    return {"a": a.detach(), "logits": logits.detach(), "loss": loss.detach(),
            "grads": {k: v.grad for k, v in p.items()}}


def folded(params, x, T, H, labels):
    """The same quantities through the fold: ybar_h = sum_n p y_n from the scores (uh g1) . kt_h, the head above the
    pooling by autograd, the token pass and the query backward by hand, as csrc/attentive.cu computes them."""
    p = {k: v.detach().clone().double() for k, v in params.items()}
    x = x.double()
    B, N, D = x.shape
    P, dh = N // T, D // H
    sc = 1 / math.sqrt(dh)
    q = p["Wq"] @ p["q0"] + p["bq"]
    kt = torch.stack([p["Wk"][h * dh:(h + 1) * dh].T @ q[h * dh:(h + 1) * dh] for h in range(H)]) * sc     # [H, D]
    u = x + p["e"].repeat_interleave(P, 0)[None]
    mu = u.mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(((u - mu) ** 2).mean(-1, keepdim=True) + EPS)
    uh = (u - mu) * rstd
    y = uh * p["g1"] + p["b1"]
    s = torch.einsum("bnd,hd->bnh", uh * p["g1"], kt)
    pr = s.softmax(1)
    ybar = torch.einsum("bnh,bnd->bhd", pr, y)
    # the head above the pooling, by autograd
    post = {k: p[k].clone().requires_grad_(True) for k in ("Wv", "bv", "Wo", "bo", "q0", "g2", "b2", "W1", "bf1",
                                                            "W2", "bf2", "Wc", "bc")}
    yb = ybar.clone().requires_grad_(True)
    a = torch.cat([yb[:, h] @ post["Wv"][h * dh:(h + 1) * dh].T for h in range(H)], 1) + post["bv"]
    z = post["q0"] + F.linear(a, post["Wo"], post["bo"])
    logits, loss = _head(post, z, labels)
    loss.backward()
    dyb = yb.grad
    # the token pass's backward (d3_atp_pool_bwd)
    c = (ybar * dyb).sum(-1)                                              # [B, H]
    dp = torch.einsum("bnd,bhd->bnh", y, dyb)
    ds = pr * (dp - c[:, None])
    dy = torch.einsum("bnh,hd->bnd", ds, kt) + torch.einsum("bnh,bhd->bnd", pr, dyb)
    gk = kt @ p["g1"]                                                     # [H]
    gd = (dyb * p["g1"]).sum(-1)                                          # [B, H]
    bd = (dyb * p["b1"]).sum(-1)
    A = (ds * gk + pr * gd[:, None]).sum(-1, keepdim=True) / D           # mean(g1 dy), from per-head scalars
    Bm = (ds * s + pr * (dp - bd[:, None])).sum(-1, keepdim=True) / D    # mean(g1 dy uh)
    du = rstd * (p["g1"] * dy - A - uh * Bm)
    grads = {k: v.grad for k, v in post.items()}
    grads["g1"] = (dy * uh).sum((0, 1))
    grads["b1"] = dy.sum((0, 1))
    grads["e"] = du.view(B, T, P, D).sum((0, 2))
    dkt = torch.einsum("bnh,bnd->hd", ds, y)
    # the query backward (d3_atp_query_bwd)
    dq = torch.cat([p["Wk"][h * dh:(h + 1) * dh] @ dkt[h] for h in range(H)]) * sc
    grads["Wk"] = torch.cat([torch.outer(q[h * dh:(h + 1) * dh], dkt[h]) for h in range(H)]) * sc
    grads["Wq"] = torch.outer(dq, p["q0"])
    grads["bq"] = dq
    grads["q0"] = grads["q0"] + p["Wq"].T @ dq
    return {"a": a.detach(), "ybar": ybar, "lse": torch.logsumexp(s, 1), "kt": kt, "logits": logits.detach(),
            "loss": loss.detach(), "grads": grads, "dybar": dyb, "dkt": dkt}
