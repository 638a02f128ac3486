"""Audio2PoseModel.infer on the library's kernels (reference src/audio_models/pose_model.py:97-124; SURVEY.md 8f N3).

  waveform -> wav2vec2 encoder on the kernels (wav2vec2.run)      -> fp16 features [T, 768] (or the sum of the 13 states)
  -> ONE ap_gemm_f16: the one-key cross-attention of every layer   -> fp32 cross [T, layers * 512]
  -> ONE ap_pose_decoder_f16: all T autoregressive steps            -> fp32 poses [T, out_dim]

The cross-attention mask leaves frame i exactly one audio frame, frame i, so layer l's cross-attention output is
out_proj(v_proj(in_fn(f_i))) for every step (pose_infer.py explains the incremental form). The three affine maps fold into
one: W_o^l W_v^l W_in and W_o^l (W_v^l b_in + b_v^l) + b_o^l, stacked over the layers into one [layers * 512, 768] GEMM,
folded in fp64 at pack time and stored as fp16 weight and fp32 bias. With `_only_last_features=False` the 1/13 of the mean
of the hidden states is folded in as well and the states are summed with ap_add_f16.

The decoder kernel gets the module's own parameters packed once (fp16 layer weights, fp32 biases, norms and pose maps), an
fp32 device copy of `biased_mask` (a plain attribute, not a buffer: `.cuda()` leaves it on the host; re-copied whenever
the attribute is replaced or modified) and of the positional table, and the identity embedding's row, chosen on the host.
There is no fallback and no torch math on the device: configurations and inputs the kernels do not cover raise before any
launch.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from .. import _lib, ops
from ..models.modeling import PackedCache, f16, f32
from . import wav2vec2

E, HEADS, FFN = ops.POSE_E, ops.POSE_HEADS, ops.POSE_FFN
MAX_OUT_DIM = 8
MAX_T = 1024     # the kernel's attention score buffer; the reference's mask and positional table stop at 600


def check_decoder(model) -> None:
    """Raises NotImplementedError naming the first property of `model` outside the geometry the decoder kernel runs."""
    dec = model.transformer_decoder
    layers = list(dec.layers)
    if not layers:
        raise NotImplementedError("pose decoder kernel: the decoder has no layers")
    if dec.norm is not None:
        raise NotImplementedError("pose decoder kernel: a final decoder norm is not supported (the reference has none)")
    eps = layers[0].norm1.eps
    for i, l in enumerate(layers):
        sa, ca = l.self_attn, l.multihead_attn
        if getattr(l, "norm_first", False):
            raise NotImplementedError(f"pose decoder kernel: layer {i} is norm_first (only post-norm is supported)")
        if not (l.activation is F.relu or isinstance(l.activation, nn.ReLU)):
            raise NotImplementedError(f"pose decoder kernel: layer {i} activation {l.activation!r} is not ReLU")
        if sa.embed_dim != E or sa.num_heads != HEADS or l.linear1.out_features != FFN:
            raise NotImplementedError(f"pose decoder kernel: layer {i} has E = {sa.embed_dim}, {sa.num_heads} heads, FFN "
                                      f"{l.linear1.out_features} (only E = {E}, {HEADS} heads, FFN {FFN})")
        for m in (sa, ca):
            if m.in_proj_weight is None or m.in_proj_bias is None or m.out_proj.bias is None:
                raise NotImplementedError(f"pose decoder kernel: layer {i} attention needs packed in_proj weights and biases")
        for lin in (l.linear1, l.linear2):
            if lin.bias is None:
                raise NotImplementedError(f"pose decoder kernel: layer {i} feed-forward without bias")
        for n in (l.norm1, l.norm2, l.norm3):
            if n.weight is None or n.bias is None or n.eps != eps:
                raise NotImplementedError(f"pose decoder kernel: layer {i} LayerNorms must be affine with one eps")
    od = model.out_dim
    if not 1 <= od <= MAX_OUT_DIM or model.pose_map_r.out_features != od or model.pose_map.in_features != od:
        raise NotImplementedError(f"pose decoder kernel: out_dim = {od} (only 1 .. {MAX_OUT_DIM})")
    if model.pose_map.out_features != E or model.in_fn.out_features != E:
        raise NotImplementedError(f"pose decoder kernel: latent_dim must be {E}")
    mask = model.biased_mask
    if mask.dim() != 3 or mask.shape[0] != HEADS or mask.shape[1] != mask.shape[2]:
        raise NotImplementedError(f"pose decoder kernel: biased_mask {tuple(mask.shape)} is not [{HEADS}, n, n]")


def fold_cross(model, only_last: bool, n_states: int):
    """The per-layer one-key cross-attention as one affine map of the encoder features, in fp32:
    (W [layers * 512, H], b [layers * 512]) with rows l * 512 .. of W f + b = out_proj_l(v_proj_l(in_fn(f))) for
    only_last, or that of the mean when f is the sum of the n_states hidden states."""
    w_in = model.in_fn.weight.detach().double()
    b_in = model.in_fn.bias.detach().double()
    if not only_last:
        w_in = w_in / n_states
    ws, bs = [], []
    for l in model.transformer_decoder.layers:
        ca = l.multihead_attn
        w_v, b_v = ca.in_proj_weight.detach()[2 * E:].double(), ca.in_proj_bias.detach()[2 * E:].double()
        w_o, b_o = ca.out_proj.weight.detach().double(), ca.out_proj.bias.detach().double()
        ws.append(w_o @ w_v @ w_in)
        bs.append(w_o @ (w_v @ b_in + b_v) + b_o)
    return torch.cat(ws).float(), torch.cat(bs).float()


def pack_decoder(model, only_last: bool, n_states: int) -> dict:
    """fp16 stacked layer weights, the fp32 per-layer vector (ops.POSE_VEC layout), the fp32 pose maps and identity table,
    and the folded cross-attention GEMM operands."""
    layers = list(model.transformer_decoder.layers)
    vec = []
    for l in layers:
        sa = l.self_attn
        vec.append(torch.cat([sa.in_proj_bias, sa.out_proj.bias, l.linear1.bias, l.linear2.bias, l.norm1.weight,
                              l.norm1.bias, l.norm2.weight, l.norm2.bias, l.norm3.weight, l.norm3.bias]).detach().float())
    cw, cb = fold_cross(model, only_last, n_states)
    return dict(
        layers=dict(w_qkv=f16(torch.stack([l.self_attn.in_proj_weight for l in layers])),
                    w_out=f16(torch.stack([l.self_attn.out_proj.weight for l in layers])),
                    w_ff1=f16(torch.stack([l.linear1.weight for l in layers])),
                    w_ff2=f16(torch.stack([l.linear2.weight for l in layers])),
                    vec=torch.stack(vec).contiguous()),
        eps=float(layers[0].norm1.eps),
        pose_map_w=f32(model.pose_map.weight), pose_map_b=f32(model.pose_map.bias),
        pose_map_r_w=f32(model.pose_map_r.weight), pose_map_r_b=f32(model.pose_map_r.bias),
        id_w=f32(model.id_embed.weight), cross_w=f16(cw), cross_b=f32(cb))


def _id_index(model, id_seed) -> int:
    """The identity row, validated as nn.Embedding would (one host read per chunk)."""
    if id_seed is None:
        raise TypeError("Audio2PoseModel.infer needs id_seed (an index tensor for id_embed), got None")
    if not isinstance(id_seed, torch.Tensor) or id_seed.is_floating_point() or id_seed.is_complex():
        raise TypeError(f"id_seed must be an integer tensor, got {type(id_seed).__name__}"
                        + (f" of {id_seed.dtype}" if isinstance(id_seed, torch.Tensor) else ""))
    if id_seed.numel() != 1:
        raise NotImplementedError(f"pose decoder kernel: batch {id_seed.numel()} is not supported (one clip per call)")
    idx = int(id_seed.reshape(-1)[0].item())
    n = model.id_embed.num_embeddings
    if not 0 <= idx < n:
        raise IndexError(f"id_seed {idx} is out of range for id_embed with {n} rows")
    return idx


class PoseDecoder:
    """Runs the decoder of one Audio2PoseModel instance on the kernels; packs on first use, re-packs when a parameter, the
    `biased_mask` attribute or the positional table changes."""

    def __init__(self, model):
        self.model = model
        self._params = {True: PackedCache(), False: PackedCache()}   # by _only_last_features: the cross fold differs
        self._aux_key = None
        self._aux = None

    def _tables(self, device):
        """fp32 device copies of the mask [8, n, n] and the positional table [m, 512]."""
        mask, pe = self.model.biased_mask, self.model.PPE.pe
        key = (id(mask), mask._version, mask.data_ptr(), pe.data_ptr(), pe._version, device)
        if key != self._aux_key:
            self._aux = (mask.detach().to(device, torch.float32).contiguous(),
                         pe.detach().reshape(-1, pe.shape[-1]).to(device, torch.float32).contiguous())
            self._aux_key = key
        return self._aux

    def _check(self, seq_len, id_seed):
        m = self.model
        check_decoder(m)
        T = int(seq_len)
        n_mask, n_pe = m.biased_mask.shape[1], m.PPE.pe.reshape(-1, m.PPE.pe.shape[-1]).shape[0]
        if not 1 <= T <= min(n_mask, n_pe, MAX_T):
            raise ValueError(f"seq_len={T} must be in [1, {min(n_mask, n_pe, MAX_T)}] (biased_mask covers {n_mask} "
                             f"positions, the positional table {n_pe}, the kernel {MAX_T})")
        return T, _id_index(m, id_seed)

    def _run(self, feats, T, idx, only_last, n_states):
        m = self.model
        pk = self._params[only_last].get(m, lambda: pack_decoder(m, only_last, n_states))
        mask, pe = self._tables(feats.device)
        with torch.no_grad():
            cross = ops.gemm(feats[:T], pk["cross_w"], bias=pk["cross_b"], out_f32=True)
            out = ops.pose_decoder(pk["layers"], pk["pose_map_w"], pk["pose_map_b"], pk["pose_map_r_w"],
                                   pk["pose_map_r_b"], pe, mask, pk["id_w"][idx], cross, T, pk["eps"])
        return out.unsqueeze(0)

    def decode(self, features: torch.Tensor, seq_len, id_seed) -> torch.Tensor:
        """The decoder alone, from the fp16 encoder features [1, S, H] or [S, H] (S >= seq_len) that in_fn reads (the
        last hidden state; with `_only_last_features=False` the SUM of the hidden states) -> fp32 [1, seq_len, out_dim]."""
        T, idx = self._check(seq_len, id_seed)
        f = features[0] if features.dim() == 3 else features
        if features.dim() == 3 and features.shape[0] != 1:
            raise NotImplementedError(f"pose decoder kernel: batch {features.shape[0]} is not supported (one clip per call)")
        if f.dim() != 2 or f.shape[1] != self.model.in_fn.in_features:
            raise ValueError(f"features {tuple(features.shape)} are not [1, S, {self.model.in_fn.in_features}]")
        if f.shape[0] < T:
            raise ValueError(f"the features have {f.shape[0]} frames, fewer than seq_len={T}")
        if not f.is_cuda:
            raise _lib.ApError("the pose decoder kernel needs the features as a CUDA tensor (no CPU fallback)")
        if f.dtype != torch.float16 or not f.is_contiguous():
            raise ValueError("the pose decoder kernel reads fp16 contiguous features (the encoder's output)")
        only_last = bool(self.model._only_last_features)
        n_states = len(self.model.audio_encoder.encoder.layers) + 1 if not only_last else 1
        return self._run(f, T, idx, only_last, n_states)

    def infer(self, enc_cache: PackedCache, input_value, seq_len, id_seed) -> torch.Tensor:
        """Audio2PoseModel.infer(input_value, seq_len, id_seed) -> fp32 [1, seq_len, out_dim]."""
        T, idx = self._check(seq_len, id_seed)
        enc = self.model.audio_encoder
        wave = wav2vec2._waveform(input_value)
        pk = enc_cache.get(enc, lambda: wav2vec2.pack_encoder(enc))
        only_last = bool(self.model._only_last_features)
        with torch.no_grad():
            last, states = wav2vec2.run(pk, wave, T, hidden_states=not only_last)
            h = last
            if not only_last:
                for s in states[:-1]:
                    h = ops.add(h, s)
        return self._run(h, T, idx, only_last, len(pk["layers"]) + 1)
