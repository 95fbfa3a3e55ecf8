"""A float64 restatement in torch of upstream DINOv3's ConvNeXt (models/convnext.py:45-335 transcribe it; the reference
module itself cannot run, DESIGN.md §2), on the reference's params tree and NHWC images, plus a random upstream-named
state dict.  Used by test_convnext_cpu.py (against Hugging Face's DINOv3ConvNextModel) and test_convnext_gpu.py."""
import torch
import torch.nn.functional as F

EPS = 1e-6


def _ln(x, w, b):
    return F.layer_norm(x, (x.shape[-1],), w.to(x.dtype), b.to(x.dtype), EPS)


def _conv(x, k, b, stride=1, padding=0, groups=1):
    """NHWC x, HWIO kernel."""
    y = F.conv2d(x.permute(0, 3, 1, 2), k.to(x.dtype).permute(3, 2, 0, 1), b.to(x.dtype), stride=stride, padding=padding,
                 groups=groups)
    return y.permute(0, 2, 3, 1)


def downsample(tree, i, x):
    d = tree[f"downsample_layers_{i}"]
    if i == 0:
        x = _conv(x, d["layers_0"]["kernel"], d["layers_0"]["bias"], stride=4)
        return _ln(x, d["layers_1"]["weight"], d["layers_1"]["bias"])
    x = _ln(x, d["layers_0"]["weight"], d["layers_0"]["bias"])
    return _conv(x, d["layers_1"]["kernel"], d["layers_1"]["bias"], stride=2)


def block(p, x):
    C = x.shape[-1]
    y = _conv(x, p["dwconv"]["kernel"], p["dwconv"]["bias"], padding=3, groups=C)
    y = _ln(y, p["norm"]["weight"], p["norm"]["bias"])
    y = F.gelu(y @ p["pwconv1"]["kernel"].to(x.dtype) + p["pwconv1"]["bias"].to(x.dtype))
    y = y @ p["pwconv2"]["kernel"].to(x.dtype) + p["pwconv2"]["bias"].to(x.dtype)
    return x + p["gamma"].to(x.dtype) * y


def stages(tree, x, last: int = 3):
    """NHWC image -> the NHWC output of every stage 0..last."""
    outs = []
    for i in range(last + 1):
        x = downsample(tree, i, x)
        s = tree[f"stages_{i}"]
        for j in range(len(s)):
            x = block(s[f"layers_{j}"], x)
        outs.append(x)
    return outs


def forward_features(tree, x):
    x = stages(tree, x)[-1]
    n, h, w, C = x.shape
    tokens = x.reshape(n, h * w, C)
    xn = _ln(torch.cat([x.mean(dim=(1, 2))[:, None], tokens], dim=1), tree["norm"]["scale"], tree["norm"]["bias"])
    return {"x_norm_clstoken": xn[:, 0], "x_storage_tokens": xn[:, 1:1], "x_norm_patchtokens": xn[:, 1:],
            "x_prenorm": tokens}


def intermediate_layers(tree, x, n=1, *, patch_size=None, reshape=False, return_class_token=False, norm=True):
    """Upstream get_intermediate_layers: per selected stage i the pooled class token of its map and its tokens (resized
    bilinearly with antialiasing to (H/p, W/p) when patch_size is set), the final norm applied when i == 3 and norm."""
    H, W = x.shape[1:3]
    take = list(range(4 - n, 4)) if isinstance(n, int) else list(n)
    maps = stages(tree, x, max(take))
    out = []
    for i in take:
        m = maps[i]
        cls = m.mean(dim=(1, 2))
        pt = m.permute(0, 3, 1, 2)
        if patch_size is not None:
            pt = F.interpolate(pt, size=(H // patch_size, W // patch_size), mode="bilinear", antialias=True)
        B, C, h, w = pt.shape
        tok = pt.flatten(2).transpose(1, 2)
        if norm and i == 3:
            cls, tok = _ln(cls, tree["norm"]["scale"], tree["norm"]["bias"]), _ln(tok, tree["norm"]["scale"], tree["norm"]["bias"])
        if reshape:
            tok = tok.transpose(1, 2).reshape(B, C, h, w)
        out.append((tok, cls))
    return tuple(out) if return_class_token else tuple(t for t, _ in out)


def upstream_state_dict(depths, dims, seed, dtype=torch.float64):
    """Random weights under upstream's names, with every LayerScale gamma in [0.1, 1] (at the 1e-6 init every block
    is close to the identity and a wrong block would go unnoticed), and upstream's `norms.3.*` alias."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g, dtype=dtype) * scale
    sd = {"downsample_layers.0.0.weight": r(dims[0], 3, 4, 4, scale=48 ** -0.5), "downsample_layers.0.0.bias": r(dims[0], scale=0.1),
          "downsample_layers.0.1.weight": 1 + r(dims[0], scale=0.1), "downsample_layers.0.1.bias": r(dims[0], scale=0.1)}
    for i in range(1, 4):
        sd[f"downsample_layers.{i}.0.weight"] = 1 + r(dims[i - 1], scale=0.1)
        sd[f"downsample_layers.{i}.0.bias"] = r(dims[i - 1], scale=0.1)
        sd[f"downsample_layers.{i}.1.weight"] = r(dims[i], dims[i - 1], 2, 2, scale=(4 * dims[i - 1]) ** -0.5)
        sd[f"downsample_layers.{i}.1.bias"] = r(dims[i], scale=0.1)
    for i in range(4):
        C = dims[i]
        for j in range(depths[i]):
            b = f"stages.{i}.{j}."
            sd[b + "gamma"] = 0.1 + 0.9 * torch.rand(C, generator=g, dtype=dtype)
            sd[b + "dwconv.weight"] = r(C, 1, 7, 7, scale=1 / 7)
            sd[b + "dwconv.bias"] = r(C, scale=0.1)
            sd[b + "norm.weight"] = 1 + r(C, scale=0.1)
            sd[b + "norm.bias"] = r(C, scale=0.1)
            sd[b + "pwconv1.weight"] = r(4 * C, C, scale=C ** -0.5)
            sd[b + "pwconv1.bias"] = r(4 * C, scale=0.1)
            sd[b + "pwconv2.weight"] = r(C, 4 * C, scale=(4 * C) ** -0.5)
            sd[b + "pwconv2.bias"] = r(C, scale=0.1)
    sd["norm.weight"], sd["norm.bias"] = 1 + r(dims[3], scale=0.1), r(dims[3], scale=0.1)
    sd["norms.3.weight"], sd["norms.3.bias"] = sd["norm.weight"].clone(), sd["norm.bias"].clone()
    return sd
