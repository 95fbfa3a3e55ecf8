"""Attentive-probe video classification of a frozen backbone: this project's own protocol, modelled on V-JEPA's
single-block attentive probe (`AttentivePooler` + linear classifier).  No published recipe or number is reproduced.

Input tokens.  Every frame of a clip goes through the backbone; the last block's normalised patch tokens
(`get_intermediate_layers(n=1, out_dtype=bf16)`) of the clip's T frames, frame after frame, make N = T * P tokens x_n
of width D.

Probe (H heads, H the backbone's head count, dh = D / H, LayerNorm eps 1e-6, MLP ratio 4):
    u_n = x_n + e_{t(n)}                          e: a learnable temporal embedding [T, D]
    y_n = LN1(u_n),  q = Wq q0 + bq               q0: the learnable query [D]
    p_{.,h} = softmax_n(q_h . (Wk y_n)_h / sqrt(dh)),  a_h = sum_n p_{n,h} (Wv y_n + bv)_h     (no key bias)
    z = q0 + Wo a + bo,  z <- z + fc2(GELU_erf(fc1(LN2(z)))),  logits = Wc z + bc
The keys fold into the query and the values out of the sum (csrc/attentive.cu): kt_h = Wk_h^T q_h / sqrt(dh) and
a_h = Wv_h ybar_h + bv_h with ybar_h = sum_n p_{n,h} y_n, so one pass over the tokens (d3_atp_pool_fwd) and one for the
backward (d3_atp_pool_bwd) replace the [N, 2D] keys and values and their gradients.  q, kt and their gradients stay in
fp32 (d3_atp_query_fwd / _bwd); everything else runs on the [B, D] rows through d3_gemm_bf16 (bf16 operands, fp32
accumulation), d3_layernorm_fwd / d3_layernorm_bwd_ls, the gelu_erf epilogue, d3_linear_xent_fwd_bwd, the column sums
and d3_adamw_ema.

Initialisation: every Linear weight, q0 and e truncated normal (std 0.02, cut at +-2), drawn in that order (q0, e, Wq,
Wk, Wv, Wo, fc1, fc2, classifier) from a CPU generator seeded with `seed`; biases 0, LayerNorm scales 1 and biases 0.
Training: cross-entropy, AdamW (0.9, 0.999, eps 1e-8) with weight decay on the 2-D parameters (the Linear weights and
e), a linear warm-up over `warmup_epochs` and a cosine decay to 0 over `epochs` passes of the train list.  Every value of
`learning_rates` trains its own probe, from the same initial weights, on the same clips; the best val top-1 wins (ties
to the first).

Clips: `num_frames` frames `frame_step` apart; an index past a video's end is its last frame.  Train: a random start in
[0, max(F - span, 0)] (span = (num_frames - 1) * frame_step + 1), one RandomResizedCrop box (scale 0.3-1, ratio
3/4-4/3) and one flip for all frames of the clip (d3_train_resized_crop per frame).  Every draw of a train clip comes
from a generator seeded by (seed, iteration, slot in the batch), so the result does not depend on `num_workers` or on
which worker decoded what.  Val: `num_segments` evenly spaced starts round(s * max(F - span, 0) / (num_segments - 1))
(the middle one when num_segments is 1) x `num_views` square boxes of the short side spread evenly along the long side
(left / centre / right for 3), each resized to `crop_size`; a video's prediction is the mean of its clips' softmax.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .. import ops
from ..engine.params import SEG_DTYPE
from .knn import RGB_MEAN, RGB_STD, _device
from .linear import K_ALIGN, InfiniteBatchSampler, sample_crop_box

bf16, f32 = torch.bfloat16, torch.float32
LEARNING_RATES = (1e-4, 3e-4, 1e-3)
TRAIN_SCALE, TRAIN_RATIO = (0.3, 1.0), (3.0 / 4.0, 4.0 / 3.0)
MLP_RATIO = 4
MAX_DIM = 1536          # d3_layernorm_bwd_ls (LN2's backward) stops at D = 1536


def probe_name(lr: float) -> str:
    return f"probe_lr_{lr:.5f}".replace(".", "_")


def clip_span(num_frames: int, frame_step: int) -> int:
    return (int(num_frames) - 1) * int(frame_step) + 1


def clip_indices(n_frames: int, start: int, num_frames: int, frame_step: int) -> list:
    """The frame indices of a clip starting at `start`, clamped to the video's last frame."""
    last = max(int(n_frames) - 1, 0)
    return [min(int(start) + i * int(frame_step), last) for i in range(int(num_frames))]


def val_clip_starts(n_frames: int, num_frames: int, frame_step: int, num_segments: int) -> list:
    """`num_segments` evenly spaced starts over [0, max(F - span, 0)]; the middle one for a single segment."""
    room = max(int(n_frames) - clip_span(num_frames, frame_step), 0)
    if int(num_segments) == 1:
        return [room // 2]
    return [int(round(s * room / (int(num_segments) - 1))) for s in range(int(num_segments))]


def view_boxes(height: int, width: int, num_views: int) -> list:
    """`num_views` square boxes (top, left, S, S) of the short side S, spread evenly along the long side (left / centre
    / right for 3 views of a landscape frame); the centre box for a single view."""
    H, W = int(height), int(width)
    S, room = min(H, W), max(H, W) - min(H, W)
    offs = [room // 2] if int(num_views) == 1 else [int(round(v * room / (int(num_views) - 1)))
                                                    for v in range(int(num_views))]
    return [(o, 0, S, S) if H > W else (0, o, S, S) for o in offs]


def clip_generator(seed: int, iteration: int, slot: int) -> torch.Generator:
    """The generator of train clip `slot` of `iteration`: a function of the three numbers only."""
    state = np.random.SeedSequence([int(seed), int(iteration), int(slot)]).generate_state(2, np.uint32)
    return torch.Generator().manual_seed(int(state[0]) << 31 ^ int(state[1]))


def sample_train_clip(seed: int, iteration: int, slot: int, n_frames: int, num_frames: int, frame_step: int):
    """(frame indices, gen): the clip's start drawn first from `clip_generator`; the caller draws the crop box and the
    flip from the returned generator once the frame size is known (`sample_train_box`)."""
    gen = clip_generator(seed, iteration, slot)
    room = max(int(n_frames) - clip_span(num_frames, frame_step), 0)
    start = int(torch.randint(0, room + 1, (1,), generator=gen).item())
    return clip_indices(n_frames, start, num_frames, frame_step), gen


def sample_train_box(gen: torch.Generator, height: int, width: int) -> tuple:
    """(top, left, h, w, flip): RandomResizedCrop(scale 0.3-1, ratio 3/4-4/3), then the flip, drawn from `gen`."""
    box = sample_crop_box(gen, int(height), int(width), scale=TRAIN_SCALE, ratio=TRAIN_RATIO)
    return box + (int(torch.rand(1, generator=gen).item() < 0.5),)


def probe_lr(lr0: float, it: int, total: int, warmup: int) -> float:
    """Linear warm-up to lr0 over `warmup` iterations, then a cosine decay to 0 at `total`."""
    if it < warmup:
        return lr0 * (it + 1) / warmup
    return lr0 * 0.5 * (1.0 + math.cos(math.pi * (it - warmup) / max(total - warmup, 1)))


class AttentiveProbe:
    """One attentive probe (see the module docstring) over clips of `num_frames` frames of P tokens of width
    `embed_dim`, trained on batches of up to `batch_size` clips for `iterations` steps.

    Parameters live in one flat fp32 buffer for d3_adamw_ema: [Wq | Wk | Wv | Wo | fc1 | fc2 | classifier | e] (weight
    decay, the matrices with bf16 copies for the GEMMs) then [q0 | g1 | b1 | bq | bv | bo | g2 | b2 | b_fc1 | b_fc2 |
    b_cls] (no decay).  The classes are padded to Cp = a multiple of 8 rows, which stay zero."""

    def __init__(self, embed_dim: int, num_heads: int, num_frames: int, num_classes: int, batch_size: int,
                 iterations: int, *, lr: float = 1e-3, weight_decay: float = 0.01, warmup_iterations: int = 0,
                 seed: int = 0, device=None):
        D, H, T, C, B = int(embed_dim), int(num_heads), int(num_frames), int(num_classes), int(batch_size)
        if D > MAX_DIM:
            raise NotImplementedError(f"attentive probe: embed_dim {D} is wider than {MAX_DIM}, the widest LayerNorm "
                                      "backward (d3_layernorm_bwd_ls) of the probe's MLP block")
        if D < 8 or D % 8 or H < 1 or D % H or (D // H) % 8:
            raise ValueError(f"embed_dim {D} must be a positive multiple of 8 split into {H} heads of a multiple of 8")
        if not 2 <= C <= 32768:
            raise ValueError("num_classes must be in [2, 32768]")
        if T < 1 or B < 1 or int(iterations) < 1:
            raise ValueError("num_frames, batch_size and iterations must be positive")
        dev = _device(device)
        self.D, self.H, self.T, self.num_classes, self.batch_size = D, H, T, C, B
        self.iterations, self.lr, self.weight_decay = int(iterations), float(lr), float(weight_decay)
        self.warmup = int(warmup_iterations)
        self.Cp = Cp = -(-C // 8) * 8
        self.device = dev
        F = MLP_RATIO * D
        mats = [("Wq", (D, D)), ("Wk", (D, D)), ("Wv", (D, D)), ("Wo", (D, D)), ("W1", (F, D)), ("W2", (D, F)),
                ("Wc", (Cp, D))]
        decayed = mats + [("e", (T, D))]
        vecs = [("q0", (D,)), ("g1", (D,)), ("b1", (D,)), ("bq", (D,)), ("bv", (D,)), ("bo", (D,)), ("g2", (D,)),
                ("b2", (D,)), ("bf1", (F,)), ("bf2", (D,)), ("bc", (Cp,))]
        offs, n = {}, 0
        for name, shape in decayed + vecs:
            offs[name] = (n, shape)
            n += int(np.prod(shape))
        self.n_mats = offs["e"][0]
        self.n_decay = offs["q0"][0]
        host = torch.zeros(n)
        gen = torch.Generator().manual_seed(int(seed))

        def draw(name, rows=None):
            o, shape = offs[name]
            t = torch.empty(shape if rows is None else (rows,) + tuple(shape[1:]))
            torch.nn.init.trunc_normal_(t, std=0.02, a=-2.0, b=2.0, generator=gen)
            host[o:o + t.numel()] = t.reshape(-1)

        for name in ("q0", "e", "Wq", "Wk", "Wv", "Wo", "W1", "W2"):
            draw(name)
        draw("Wc", rows=C)
        for name in ("g1", "g2"):
            o, shape = offs[name]
            host[o:o + shape[0]] = 1.0
        self.p = host.to(dev)
        self.g, self.m, self.v = (torch.zeros(n, dtype=f32, device=dev) for _ in range(3))
        view = lambda buf, name: buf[offs[name][0]:offs[name][0] + int(np.prod(offs[name][1]))].view(offs[name][1])
        self.params = {name: view(self.p, name) for name in offs}
        self.grads = {name: view(self.g, name) for name in offs}
        self.p_bf16 = torch.empty(self.n_mats, dtype=bf16, device=dev)
        ops.cast_f32_bf16(self.p[:self.n_mats], self.p_bf16)
        self.w16 = {name: self.p_bf16[offs[name][0]:offs[name][0] + int(np.prod(shape))].view(shape)
                    for name, shape in mats}
        # the kernel's EMA operands: at momentum 1 they keep their values, nothing reads them
        self._ema, self._ema_bf16 = torch.zeros(n, dtype=f32, device=dev), torch.zeros(self.n_mats, dtype=bf16, device=dev)
        segs = np.zeros(2, dtype=SEG_DTYPE)
        segs[0] = (0, 1.0, 1.0, 0, 0)
        segs[1] = (self.n_decay, 1.0, 0.0, 0, 0)
        self.segs = torch.from_numpy(segs.view(np.uint8).copy()).to(dev)
        # activations; the weight-gradient GEMMs contract over the batch, padded with zero rows to whole k-blocks
        Bp = self.Bp = -(-B // K_ALIGN) * K_ALIGN
        z = lambda *shape, dtype=f32: torch.zeros(*shape, dtype=dtype, device=dev)
        self.q, self.kt, self.dkt = z(D), z(H, D), z(H, D)
        self.ybar, self.lse, self.dybar = z(B, H, D), z(B, H), z(B, H, D)
        self.ybf, self.abf, self.dabf = z(Bp, H, D, dtype=bf16), z(Bp, D, dtype=bf16), z(Bp, D, dtype=bf16)
        self.q0rows, self.zz, self.mean2, self.rstd2 = z(B, D), z(B, D), z(B), z(B)
        self.y2bf, self.h1bf, self.h1pre = z(Bp, D, dtype=bf16), z(Bp, F, dtype=bf16), z(Bp, F, dtype=bf16)
        self.z2, self.z2bf, self.logits = z(B, D), z(Bp, D, dtype=bf16), z(B, Cp)
        self.dlog, self.dz2, self.dz2bf = z(Bp, Cp, dtype=bf16), z(B, D), z(Bp, D, dtype=bf16)
        self.dh1, self.dpre, self.dy2 = z(B, F), z(Bp, F, dtype=bf16), z(B, D)
        self.dz, self.dzbf = z(B, D), z(Bp, D, dtype=bf16)
        self.loss, self.labels = z(1), torch.zeros(B, dtype=torch.int32, device=dev)
        self.steps = 0

    def _check_tokens(self, x: torch.Tensor) -> int:
        n = x.shape[0]
        if x.dtype != bf16 or x.dim() != 3 or x.shape[2] != self.D or x.shape[1] % self.T or not 1 <= n <= self.batch_size:
            raise ValueError(f"tokens must be bf16 [<= {self.batch_size}, {self.T} * P, {self.D}], got {x.dtype} "
                             f"{tuple(x.shape)}")
        return n

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """fp32 [n, Cp] logits of the clips' tokens x (bf16 [n, T * P, D]); columns >= num_classes are padding."""
        n, P_ = self._check_tokens(x), self.params
        D, H, dh, w16 = self.D, self.H, self.D // self.H, self.w16
        ops.atp_query_fwd(P_["q0"], P_["Wq"], P_["bq"], P_["Wk"], H, self.q, self.kt)
        ops.atp_pool_fwd(x.contiguous(), self.T, P_["e"], P_["g1"], P_["b1"], self.kt, self.ybar[:n], self.lse[:n])
        ops.cast_f32_bf16(self.ybar[:n], self.ybf[:n])
        for h in range(H):                   # a_h = Wv_h ybar_h + bv_h
            hs = slice(h * dh, (h + 1) * dh)
            ops.gemm(self.ybf[:n, h], w16["Wv"][hs], self.abf[:n, hs], bias=P_["bv"][hs])
        self.q0rows[:n].copy_(P_["q0"].expand(n, D))
        ops.gemm(self.abf[:n], w16["Wo"], self.zz[:n], bias=P_["bo"], resid=self.q0rows[:n])
        ops.layernorm_fwd(self.zz[:n], P_["g2"], P_["b2"], self.y2bf[:n], self.mean2[:n], self.rstd2[:n])
        ops.gemm(self.y2bf[:n], w16["W1"], self.h1bf[:n], bias=P_["bf1"], gelu_erf=True, store_pre=self.h1pre[:n])
        ops.gemm(self.h1bf[:n], w16["W2"], self.z2[:n], bias=P_["bf2"], resid=self.zz[:n])
        ops.cast_f32_bf16(self.z2[:n], self.z2bf[:n])
        return ops.gemm(self.z2bf[:n], w16["Wc"], self.logits[:n], bias=P_["bc"])

    def gradients(self, x: torch.Tensor, labels) -> torch.Tensor:
        """The batch-mean cross-entropy of the clips x (bf16 [B, T * P, D], B = batch_size) against `labels` and its
        gradient into self.g (every parameter).  Returns the device fp32 [1] loss (no host sync)."""
        B = self._check_tokens(x)
        if B != self.batch_size:
            raise ValueError(f"a train batch has {self.batch_size} clips, got {B}")
        y = torch.as_tensor(labels).reshape(-1)
        if y.numel() != B:
            raise ValueError(f"{y.numel()} labels for a batch of {B}")
        self.labels.copy_(y)
        self.forward(x)
        P_, G, w16 = self.params, self.grads, self.w16
        H, dh = self.H, self.D // self.H
        ops.linear_xent_fwd_bwd(self.logits, self.labels, self.num_classes, self.Cp, self.loss, self.dlog)
        ops.gemm(self.dlog, self.z2bf, G["Wc"], a_mn=True, b_mn=True)
        for name in ("bc", "bf2", "bf1", "bo", "bv", "q0", "g2", "b2"):
            G[name].zero_()
        ops.colsum_bf16(self.dlog[:B], G["bc"])
        ops.gemm(self.dlog[:B], w16["Wc"], self.dz2, b_mn=True)
        ops.cast_f32_bf16(self.dz2, self.dz2bf[:B])
        ops.gemm(self.dz2bf, self.h1bf, G["W2"], a_mn=True, b_mn=True)
        ops.colsum_bf16(self.dz2bf[:B], G["bf2"])
        ops.gemm(self.dz2bf[:B], w16["W2"], self.dh1, b_mn=True)
        ops.atp_gelu_erf_bwd(self.dh1, self.h1pre[:B], self.dpre[:B])
        ops.gemm(self.dpre, self.y2bf, G["W1"], a_mn=True, b_mn=True)
        ops.colsum_bf16(self.dpre[:B], G["bf1"])
        ops.gemm(self.dpre[:B], w16["W1"], self.dy2, b_mn=True)
        ops.layernorm_bwd_ls(self.dy2, self.zz, self.mean2, self.rstd2, P_["g2"], self.dz, dx_add=self.dz2,
                             dscale=G["g2"], dbias=G["b2"])
        ops.cast_f32_bf16(self.dz, self.dzbf[:B])
        ops.gemm(self.dzbf, self.abf, G["Wo"], a_mn=True, b_mn=True)
        ops.colsum_bf16(self.dzbf[:B], G["bo"])
        ops.colsum_f32(self.dz, G["q0"])                 # z = q0 + ...: q0 is shared by the clips
        ops.gemm(self.dzbf[:B], w16["Wo"], self.dabf[:B], b_mn=True)
        ops.colsum_bf16(self.dabf[:B], G["bv"])
        for h in range(H):
            hs = slice(h * dh, (h + 1) * dh)
            ops.gemm(self.dabf[:, hs], self.ybf[:, h], G["Wv"][hs], a_mn=True, b_mn=True)
            ops.gemm(self.dabf[:B, hs], w16["Wv"][hs], self.dybar[:, h], b_mn=True)
        ops.atp_pool_bwd(x.contiguous(), self.T, P_["e"], P_["g1"], P_["b1"], self.kt, self.lse, self.ybar, self.dybar,
                         self.dkt, G["g1"], G["b1"], G["e"])
        ops.atp_query_bwd(P_["q0"], P_["Wq"], P_["Wk"], self.q, self.dkt, G["Wq"], G["bq"], G["Wk"], G["q0"])
        return self.loss

    def step(self, x: torch.Tensor, labels, it: int) -> torch.Tensor:
        """One AdamW step on a batch of clips at schedule iteration `it`; returns the device fp32 [1] loss."""
        loss = self.gradients(x, labels)
        self.steps += 1
        lr = probe_lr(self.lr, int(it), self.iterations, self.warmup)
        ops.adamw_ema(self.p, self.g, self.m, self.v, self._ema, self.p_bf16, self._ema_bf16, self.n_mats, self.segs, 2,
                      None, 0.0, lr, lr, self.weight_decay, self.steps, 1.0)
        return loss

    def state_dict(self) -> dict:
        """{name: fp32 tensor} on the host (the classifier without its padding rows)."""
        C = self.num_classes
        out = {k: v.cpu().clone() for k, v in self.params.items()}
        out["Wc"], out["bc"] = out["Wc"][:C].clone(), out["bc"][:C].clone()
        return out


class _TrainClips:
    """Train clip (idx, iteration, slot) of a video dataset: frames uint8 [T, H, W, 3], label, box (top, left, h, w,
    flip); every draw from `clip_generator(seed, iteration, slot)`."""

    def __init__(self, dataset, num_frames: int, frame_step: int, seed: int):
        self.dataset, self.num_frames, self.frame_step, self.seed = dataset, int(num_frames), int(frame_step), int(seed)

    def __getitem__(self, key):
        idx, it, slot = key
        n = self.dataset.frame_count(idx)
        indices, gen = sample_train_clip(self.seed, it, slot, n, self.num_frames, self.frame_step)
        frames = self.dataset.load_frames(idx, indices)
        return frames, int(self.dataset.targets[idx]), sample_train_box(gen, frames.shape[1], frames.shape[2])


class _ClipBatches:
    """[(idx, iteration, slot)] per iteration, the indices from InfiniteBatchSampler."""

    def __init__(self, n: int, batch_size: int, iterations: int, seed: int):
        self.sampler = InfiniteBatchSampler(n, batch_size, iterations, seed)

    def __len__(self):
        return len(self.sampler)

    def __iter__(self):
        for it, batch in enumerate(self.sampler):
            yield [(i, it, s) for s, i in enumerate(batch)]


class _ValClips:
    """Val video i: frames uint8 [num_segments * T, H, W, 3] (segment after segment), its label."""

    def __init__(self, dataset, num_frames: int, frame_step: int, num_segments: int):
        self.dataset, self.num_frames, self.frame_step = dataset, int(num_frames), int(frame_step)
        self.num_segments = int(num_segments)

    def __len__(self):
        return len(self.dataset)

    def __getitem__(self, i):
        n = self.dataset.frame_count(i)
        idx = [j for s in val_clip_starts(n, self.num_frames, self.frame_step, self.num_segments)
               for j in clip_indices(n, s, self.num_frames, self.frame_step)]
        return self.dataset.load_frames(i, idx), int(self.dataset.targets[i])


def _pack_frames(frames_list):
    """Frames of several clips -> (flat uint8, desc int64 [n, 3] = (offset, H, W)), frame after frame."""
    frames = [np.ascontiguousarray(f, dtype=np.uint8) for f in frames_list]
    for f in frames:
        if f.ndim != 4 or f.shape[3] != 3:
            raise ValueError(f"expected uint8 frames [T, H, W, 3], got shape {f.shape}")
    desc, off = [], 0
    for f in frames:
        for _ in range(f.shape[0]):
            desc.append((off, f.shape[1], f.shape[2]))
            off += f.shape[1] * f.shape[2] * 3
    flat = torch.from_numpy(np.concatenate([f.reshape(-1) for f in frames]))
    return flat, torch.tensor(desc, dtype=torch.int64).reshape(-1, 3)


def _collate_train(batch):
    flat, desc = _pack_frames([f for f, _, _ in batch])
    T = batch[0][0].shape[0]
    boxes = torch.tensor([b for _, _, b in batch for _ in range(T)], dtype=torch.int32).reshape(-1, 5)
    return flat, desc, torch.tensor([y for _, y, _ in batch], dtype=torch.int64), boxes


def _collate_val(batch):
    flat, desc = _pack_frames([f for f, _ in batch])
    return flat, desc, torch.tensor([y for _, y in batch], dtype=torch.int64)


def clip_tokens(model, images: torch.Tensor, n_clips: int) -> torch.Tensor:
    """bf16 [n_clips, T * P, D]: the last block's normalised patch tokens of the frames [n_clips * T, S, S, 3], frame
    after frame within each clip."""
    patches = model.get_intermediate_layers(images, n=1, out_dtype=bf16)[0]
    n, P, D = patches.shape
    return patches.reshape(int(n_clips), (n // int(n_clips)) * P, D)


def _accuracies(probs: torch.Tensor, labels: torch.Tensor, C: int) -> dict:
    """top-1 / top-5 (percent) and mean per-class accuracy (percent over the classes present) of mean probabilities."""
    top = probs.topk(min(5, C), dim=1).indices.cpu()
    y = labels.cpu()
    hit1 = top[:, 0] == y
    hit5 = (top == y[:, None]).any(1)
    present = torch.unique(y)
    per_class = torch.stack([hit1[y == c].double().mean() for c in present])
    return {"top1": 100.0 * float(hit1.double().mean()), "top5": 100.0 * float(hit5.double().mean()),
            "mean_per_class": 100.0 * float(per_class.mean())}


def eval_attentive(model, train_dataset, val_dataset, *, learning_rates=LEARNING_RATES, epochs: int = 20,
                   warmup_epochs: int = 0, weight_decay: float = 0.01, batch_size: int = 16, num_frames: int = 16,
                   frame_step: int = 4, num_segments: int = 2, num_views: int = 3, crop_size: int = 224,
                   num_workers: int = 8, seed: int = 0, rgb_mean=RGB_MEAN, rgb_std=RGB_STD, num_classes=None,
                   device=None, **_ignored) -> dict:
    """Train one attentive probe per learning rate on `train_dataset` and score `val_dataset` (datasets with
    `targets`, `frame_count(i)` and `load_frames(i, indices)`, see eval.datasets).  Returns {"probes": {name: {"lr",
    "top1", "top5", "mean_per_class"}}, "best_probe", "top1", "top5", "mean_per_class", and the video / clip counts}.
    The extra keys of an `evaluation.attentive` block (dataset paths) are accepted and ignored."""
    dev = _device(device if device is not None else getattr(model, "device", None))
    targets = list(train_dataset.targets) + list(val_dataset.targets)
    C = int(num_classes) if num_classes is not None else int(max(targets)) + 1
    B, T, S = int(batch_size), int(num_frames), int(crop_size)
    epoch_length = max(len(train_dataset) // B, 1)
    iterations, warmup = int(epochs) * epoch_length, int(warmup_epochs) * epoch_length
    lrs = [float(v) for v in learning_rates]
    if not lrs:
        raise ValueError("learning_rates is empty")
    D, H = int(model.embed_dim), int(model.num_heads)
    probes = [AttentiveProbe(D, H, T, C, B, iterations, lr=lr, weight_decay=weight_decay, warmup_iterations=warmup,
                             seed=seed, device=dev) for lr in lrs]
    pin = dev.type == "cuda"
    loader = torch.utils.data.DataLoader(_TrainClips(train_dataset, T, frame_step, seed),
                                         batch_sampler=_ClipBatches(len(train_dataset), B, iterations, seed),
                                         num_workers=int(num_workers), collate_fn=_collate_train, pin_memory=pin,
                                         persistent_workers=False)
    images = torch.empty(B * T, S, S, 3, dtype=bf16, device=dev)
    for it, (flat, desc, y, boxes) in enumerate(loader):
        ops.train_resized_crop(flat.to(dev, non_blocking=True), desc.to(dev, non_blocking=True), boxes.to(dev), images,
                               max_taps=ops.train_max_taps(boxes.tolist(), S), mean=rgb_mean, std=rgb_std)
        x = clip_tokens(model, images, B)
        for probe in probes:
            probe.step(x, y, it)
    K = int(num_segments) * int(num_views)
    per_batch = max(B // K, 1)
    val_loader = torch.utils.data.DataLoader(_ValClips(val_dataset, T, frame_step, num_segments), batch_size=per_batch,
                                             shuffle=False, num_workers=int(num_workers), collate_fn=_collate_val,
                                             pin_memory=pin, persistent_workers=False)
    probs = [torch.zeros(len(val_dataset), C, dtype=torch.float64, device=dev) for _ in probes]
    labels = torch.empty(len(val_dataset), dtype=torch.int64)
    v0 = 0
    for flat, desc, y in val_loader:
        nv = y.numel()
        frames_per_video = desc.shape[0] // nv
        rows, boxes = [], []
        for v in range(nv):
            base = v * frames_per_video
            H0, W0 = int(desc[base, 1]), int(desc[base, 2])
            for s in range(int(num_segments)):
                for box in view_boxes(H0, W0, num_views):
                    for t in range(T):
                        rows.append(base + s * T + t)
                        boxes.append(box + (0,))
        sel = torch.tensor(rows, dtype=torch.int64)
        bx = torch.tensor(boxes, dtype=torch.int32)
        clips = nv * K
        clip_probs = [torch.empty(clips, C, dtype=torch.float64, device=dev) for _ in probes]
        for c0 in range(0, clips, B):
            c1 = min(clips, c0 + B)
            r = slice(c0 * T, c1 * T)
            imgs = images[:(c1 - c0) * T]
            ops.train_resized_crop(flat.to(dev, non_blocking=True), desc[sel[r]].contiguous().to(dev),
                                   bx[r].contiguous().to(dev), imgs, max_taps=ops.train_max_taps(bx[r].tolist(), S),
                                   mean=rgb_mean, std=rgb_std)
            x = clip_tokens(model, imgs, c1 - c0)
            for probe, cp in zip(probes, clip_probs):
                cp[c0:c1] = torch.softmax(probe.forward(x)[:, :C].double(), dim=1)
        for pr, cp in zip(probs, clip_probs):
            pr[v0:v0 + nv] = cp.view(nv, K, C).mean(1)
        labels[v0:v0 + nv] = y
        v0 += nv
    if v0 == 0:
        raise ValueError("empty val dataset")
    results = {"probes": {}}
    for lr, pr in zip(lrs, probs):
        results["probes"][probe_name(lr)] = {"lr": lr, **_accuracies(pr, labels, C)}
    best = probe_name(lrs[0])
    for lr in lrs[1:]:
        if results["probes"][probe_name(lr)]["top1"] > results["probes"][best]["top1"]:
            best = probe_name(lr)
    results["best_probe"] = {"name": best, **results["probes"][best]}
    results.update({k: results["probes"][best][k] for k in ("top1", "top5", "mean_per_class")})
    results.update({"train_videos": len(train_dataset), "val_videos": len(val_dataset), "train_clips": iterations * B,
                    "val_clips": len(val_dataset) * K, "iterations": iterations})
    return results
