"""The wav2vec2-base audio encoder and the Audio2Mesh head on the library's sm_90a kernels (SURVEY.md 8f, N3).

The reference runs transformers' Wav2Vec2Model through a thin wrapper (src/audio_models/wav2vec2.py:30-64) in fp32 on
cuBLAS / cuDNN: once over the whole clip for Audio2MeshModel.infer and once per 5 s chunk for Audio2PoseModel.infer
(scripts/audio2vid.py:162,189-195). Here the same module's parameters are packed once to fp16 and the forward pass is:

  waveform [S] fp32 -> ap_conv1d_stem_f32 (Conv1d(1, 512, 10, 5))               -> [T0, 512]
  -> ap_batchnorm_train_nhwc_f16 with GELU       (GroupNorm(512, 512) over time == per-channel batch statistics)
  -> 6 x ap_gemm_f16 with the GELU epilogue       (Conv1d(512, 512, k in {3, 2}, stride 2) over frame pairs, no im2col)
  -> ap_resample_rows_linear_f16                  (linear_interpolation to seq_len frames, align_corners=True)
  -> ap_layernorm_f16 -> ap_gemm_f16              (feature projection 512 -> 768)
  -> ap_pos_conv1d_gelu_f16 -> ap_layernorm_f16   (x + GELU(grouped positional conv), encoder.layer_norm)
  -> 12 x [q|k|v GEMM, ap_attention_f16 (12 heads, d = 64), out GEMM + residual, LayerNorm,
           GEMM + GELU (768 -> 3072), GEMM + residual (3072 -> 768), LayerNorm]           (post-LN layers)

`enable_kernels(model)` rebinds `audio_encoder.forward` on an Audio2MeshModel / Audio2PoseModel instance (and, for
Audio2Mesh, `infer`, whose in_fn / out_fn head becomes two GEMMs); parameters, state dict and module tree are untouched.
There is no fallback: inputs or configurations the kernels do not cover raise.
"""
from __future__ import annotations

import types

import torch

from .. import _lib, ops
from ..models.modeling import PackedCache, f16, f32

# the wav2vec2-base geometry the kernels implement (transformers Wav2Vec2Config defaults, facebook/wav2vec2-base-960h)
BASE_GEOMETRY = dict(feat_extract_norm="group", do_stable_layer_norm=False, conv_bias=False,
                     conv_dim=(512,) * 7, conv_kernel=(10, 3, 3, 3, 3, 2, 2), conv_stride=(5, 2, 2, 2, 2, 2, 2),
                     feat_extract_activation="gelu", hidden_act="gelu", num_conv_pos_embeddings=128,
                     num_conv_pos_embedding_groups=16, add_adapter=False)
HEAD_DIM = 64
MIN_SAMPLES = 400    # the shortest waveform that leaves one frame after the seven convolutions


def check_config(cfg) -> None:
    """Raises NotImplementedError naming the first field where `cfg` leaves the geometry the kernels implement."""
    for field, want in BASE_GEOMETRY.items():
        got = getattr(cfg, field, None)
        if isinstance(want, tuple):
            got = tuple(got) if got is not None else None
        if got != want:
            raise NotImplementedError(f"wav2vec2 kernels: config.{field} = {got!r} is not supported (only {want!r})")
    if cfg.hidden_size % cfg.num_attention_heads or cfg.hidden_size // cfg.num_attention_heads != HEAD_DIM:
        raise NotImplementedError(f"wav2vec2 kernels: config.num_attention_heads = {cfg.num_attention_heads} gives "
                                  f"head_dim {cfg.hidden_size / cfg.num_attention_heads}, only {HEAD_DIM} is supported")
    if cfg.hidden_size != 48 * cfg.num_conv_pos_embedding_groups:
        raise NotImplementedError(f"wav2vec2 kernels: config.hidden_size = {cfg.hidden_size} is not 48 channels x "
                                  f"{cfg.num_conv_pos_embedding_groups} positional-convolution groups")


def conv_frames(samples: int) -> list:
    """Frame counts after each of the seven feature-extractor convolutions."""
    t, out = samples, []
    for k, s in zip(BASE_GEOMETRY["conv_kernel"], BASE_GEOMETRY["conv_stride"]):
        t = (t - k) // s + 1
        out.append(t)
    return out


def fold_weight_norm(conv: torch.nn.Conv1d) -> torch.Tensor:
    """The positional convolution's weight g * v / ||v|| (norm over every dim but 2), in fp32, from either storage:
    torch.nn.utils.parametrizations.weight_norm (original0 = g, original1 = v) or the older weight_g / weight_v."""
    par = getattr(conv, "parametrizations", None)
    if par is not None and "weight" in par:
        g, v = par.weight.original0, par.weight.original1
    elif hasattr(conv, "weight_g") and hasattr(conv, "weight_v"):
        g, v = conv.weight_g, conv.weight_v
    else:
        return conv.weight.detach().float()
    return torch._weight_norm(v.detach().float(), g.detach().float(), 2)


def pack_encoder(enc) -> dict:
    """fp16 kernel-layout copies of a Wav2Vec2Model's parameters (fp32 for the stem, biases and norm affines)."""
    cfg = enc.config
    fe = enc.feature_extractor.conv_layers
    gn = fe[0].layer_norm
    pk = dict(stem_w=f32(fe[0].conv.weight.reshape(fe[0].conv.weight.shape[0], -1)), gn_g=f32(gn.weight),
              gn_b=f32(gn.bias), gn_eps=float(gn.eps),
              convs=[(ops.pack_conv1d_weight(l.conv.weight.detach()), l.conv.kernel_size[0]) for l in fe[1:]])
    fp = enc.feature_projection
    pk.update(fp_ln_g=f32(fp.layer_norm.weight), fp_ln_b=f32(fp.layer_norm.bias), fp_ln_eps=float(fp.layer_norm.eps),
              fp_w=f16(fp.projection.weight), fp_b=f32(fp.projection.bias))
    pc = enc.encoder.pos_conv_embed.conv
    pk.update(pos_w=ops.pack_pos_conv_weight(fold_weight_norm(pc)), pos_b=f32(pc.bias), pos_groups=pc.groups,
              enc_ln_g=f32(enc.encoder.layer_norm.weight), enc_ln_b=f32(enc.encoder.layer_norm.bias),
              enc_ln_eps=float(enc.encoder.layer_norm.eps))
    layers = []
    for l in enc.encoder.layers:
        a, ff = l.attention, l.feed_forward
        layers.append(dict(
            qkv_w=f16(torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight])),
            qkv_b=f32(torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias])),
            out_w=f16(a.out_proj.weight), out_b=f32(a.out_proj.bias),
            ln1=(f32(l.layer_norm.weight), f32(l.layer_norm.bias), float(l.layer_norm.eps)),
            ff1_w=f16(ff.intermediate_dense.weight), ff1_b=f32(ff.intermediate_dense.bias),
            ff2_w=f16(ff.output_dense.weight), ff2_b=f32(ff.output_dense.bias),
            ln2=(f32(l.final_layer_norm.weight), f32(l.final_layer_norm.bias), float(l.final_layer_norm.eps))))
    pk["layers"] = layers
    pk["heads"] = cfg.num_attention_heads
    return pk


def run(pk: dict, wave: torch.Tensor, seq_len: int, hidden_states: bool = False):
    """The encoder on the library's kernels. wave: fp32 [S] on the device. Returns fp16 [seq_len, 768] (the
    last_hidden_state) and, with hidden_states, the list of the 13 fp16 hidden states (the last one is the first result)."""
    frames = conv_frames(wave.numel())
    if frames[-1] < 1:
        raise ValueError(f"wav2vec2: a waveform of {wave.numel()} samples leaves no frame after the feature extractor "
                         f"(at least {MIN_SAMPLES} samples are needed)")
    if seq_len < 1:
        raise ValueError(f"wav2vec2: seq_len={seq_len} must be >= 1")
    h = ops.conv1d_stem(wave, pk["stem_w"])
    h = ops.batch_norm_train(h, pk["gn_g"], pk["gn_b"], pk["gn_eps"], act="gelu")
    for w, k in pk["convs"]:
        h = ops.conv1d_s2(h, w, k, gelu=True)
    h = ops.resample_rows_linear(h, seq_len)
    h = ops.layer_norm(h, pk["fp_ln_g"], pk["fp_ln_b"], pk["fp_ln_eps"])
    h = ops.gemm(h, pk["fp_w"], bias=pk["fp_b"])
    h = ops.pos_conv1d_gelu(h, pk["pos_w"], pk["pos_b"], pk["pos_groups"])
    h = ops.layer_norm(h, pk["enc_ln_g"], pk["enc_ln_b"], pk["enc_ln_eps"])
    states = [h] if hidden_states else None
    heads = pk["heads"]
    c = h.shape[1]
    for L in pk["layers"]:
        qkv = ops.gemm(h, L["qkv_w"], bias=L["qkv_b"])
        a = ops.attention(qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:], n_frames=1, tokens=seq_len, heads=heads,
                          head_dim=HEAD_DIM, dpad=HEAD_DIM)
        x = ops.gemm(a, L["out_w"], bias=L["out_b"], residual=h)
        h = ops.layer_norm(x, *L["ln1"])
        f = ops.gemm(h, L["ff1_w"], bias=L["ff1_b"], gelu=True)
        x = ops.gemm(f, L["ff2_w"], bias=L["ff2_b"], residual=h)
        h = ops.layer_norm(x, *L["ln2"])
        if hidden_states:
            states.append(h)
    return h, states


def _waveform(input_values: torch.Tensor) -> torch.Tensor:
    """[1, S] waveform -> fp32 [S] on its device; shape, length and device are checked in that order."""
    if not isinstance(input_values, torch.Tensor) or input_values.dim() != 2:
        raise ValueError("wav2vec2: input_values must be a [batch, samples] tensor")
    if input_values.shape[0] != 1:
        raise NotImplementedError(f"wav2vec2 kernels: batch {input_values.shape[0]} is not supported (one clip per call)")
    if conv_frames(input_values.shape[1])[-1] < 1:
        raise ValueError(f"wav2vec2: a waveform of {input_values.shape[1]} samples leaves no frame after the feature "
                         f"extractor (at least {MIN_SAMPLES} samples are needed)")
    if not input_values.is_cuda:
        raise _lib.ApError("wav2vec2 kernels need the waveform as a CUDA tensor (no CPU fallback)")
    return input_values[0].to(torch.float32).contiguous()


def _check_call(attention_mask, mask_time_indices, output_attentions):
    if attention_mask is not None:
        raise NotImplementedError("wav2vec2 kernels: attention_mask is not supported (the reference's inference passes none)")
    if mask_time_indices is not None:
        raise NotImplementedError("wav2vec2 kernels: mask_time_indices is not supported")
    if output_attentions:
        raise NotImplementedError("wav2vec2 kernels: output_attentions=True is not supported (attention maps are never "
                                  "materialised)")


def _encoder_forward(enc, cache: PackedCache, input_values, seq_len, attention_mask=None, mask_time_indices=None,
                     output_attentions=None, output_hidden_states=None, return_dict=None):
    """The reference wrapper's forward signature and result, computed by run()."""
    from transformers.modeling_outputs import BaseModelOutput
    _check_call(attention_mask, mask_time_indices, output_attentions)
    wave = _waveform(input_values)
    output_hidden_states = (output_hidden_states if output_hidden_states is not None
                            else enc.config.output_hidden_states)
    return_dict = return_dict if return_dict is not None else getattr(enc.config, "return_dict", True)
    pk = cache.get(enc, lambda: pack_encoder(enc))
    with torch.no_grad():
        last, states = run(pk, wave, int(seq_len), hidden_states=bool(output_hidden_states))
    last = last.float().unsqueeze(0)
    states = tuple(s.float().unsqueeze(0) for s in states) if states is not None else None
    if not return_dict:
        return (last,) + ((states,) if states is not None else ())
    return BaseModelOutput(last_hidden_state=last, hidden_states=states, attentions=None)


def _pack_mesh_head(model, only_last: bool, n_layers: int) -> dict:
    """in_fn / out_fn as GEMM operands. With the mean of the 13 hidden states, 1/13 is folded into in_fn's weight; out_fn's
    rows are zero padded to a multiple of 64 (N = 1404 -> 1408) and the padding is never written (n_valid)."""
    w_in = model.in_fn.weight.detach().float()
    if not only_last:
        w_in = w_in / (n_layers + 1)
    w_out, b_out = model.out_fn.weight.detach().float(), model.out_fn.bias.detach().float()
    n = w_out.shape[0]
    n_pad = (n + 63) // 64 * 64
    wp = torch.zeros(n_pad, w_out.shape[1], dtype=torch.float16, device=w_out.device)
    wp[:n] = w_out.to(torch.float16)
    bp = torch.zeros(n_pad, dtype=torch.float32, device=w_out.device)
    bp[:n] = b_out
    return dict(in_w=f16(w_in), in_b=f32(model.in_fn.bias), out_w=wp.contiguous(), out_b=bp, n_out=n)


def mesh_infer(model, enc_cache: PackedCache, head_cache: PackedCache, input_value, seq_len):
    """Audio2MeshModel.infer (reference src/audio_models/model.py:58-69) -> fp32 [1, seq_len, out_dim]."""
    enc = model.audio_encoder
    only_last = bool(model._only_last_features)
    wave = _waveform(input_value)
    pk = enc_cache.get(enc, lambda: pack_encoder(enc))
    head = head_cache.get(model, lambda: _pack_mesh_head(model, only_last, len(pk["layers"])))
    with torch.no_grad():
        last, states = run(pk, wave, int(seq_len), hidden_states=not only_last)
        h = last
        if not only_last:
            for s in states[:-1]:
                h = ops.add(h, s)
        lat = ops.gemm(h, head["in_w"], bias=head["in_b"])
        out = ops.gemm(lat, head["out_w"], bias=head["out_b"], n_valid=head["n_out"], out_f32=True)
    return out.unsqueeze(0)


def enable_kernels(model):
    """Run `model.audio_encoder` and `model.infer` on the library's kernels.

    model: an instance of the reference's Audio2MeshModel (has in_fn / out_fn, no decoder: `infer` runs the in_fn / out_fn
    head as two GEMMs) or Audio2PoseModel (has transformer_decoder: `infer` runs the encoder, the folded cross-attention
    GEMM and the one-launch decoder of pose_decoder.py). Only bound methods on the instances change. For an
    Audio2PoseModel, `enable_kv_cache` also rebinds `infer`: whichever of the two was applied last decides which `infer`
    runs (the encoder stays on the kernels either way)."""
    enc = getattr(model, "audio_encoder", None)
    if enc is None or not hasattr(enc, "config"):
        raise TypeError(f"enable_kernels: {type(model).__name__} has no wav2vec2 audio_encoder")
    check_config(enc.config)
    is_pose = hasattr(model, "transformer_decoder")
    if not is_pose and not (hasattr(model, "in_fn") and hasattr(model, "out_fn")):
        raise TypeError(f"enable_kernels: {type(model).__name__} is neither an Audio2MeshModel nor an Audio2PoseModel")
    enc_cache = PackedCache()

    def forward(self, input_values, seq_len, attention_mask=None, mask_time_indices=None, output_attentions=None,
                output_hidden_states=None, return_dict=None):
        return _encoder_forward(self, enc_cache, input_values, seq_len, attention_mask, mask_time_indices,
                                output_attentions, output_hidden_states, return_dict)
    enc.forward = types.MethodType(forward, enc)

    if not is_pose:
        head_cache = PackedCache()

        def infer(self, input_value, seq_len):
            return mesh_infer(self, enc_cache, head_cache, input_value, seq_len)
    else:
        from .pose_decoder import PoseDecoder
        decoder = PoseDecoder(model)

        def infer(self, input_value, seq_len, id_seed=None):
            return decoder.infer(enc_cache, input_value, seq_len, id_seed)
    model.infer = types.MethodType(infer, model)
    return model
