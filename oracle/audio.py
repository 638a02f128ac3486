"""fp32 restatement of the reference's wav2vec2 wrapper forward (src/audio_models/wav2vec2.py:30-64) and of
Audio2MeshModel.infer (src/audio_models/model.py:58-69), built from the transformers submodules in the wrapper's order:
feature_extractor -> linear interpolation to seq_len (torch_utils.py:16-19) -> feature_projection -> encoder.
It runs on any device, so the GPU tests use it as the oracle at clip lengths whose reference outputs are too big to store;
tests/test_audio_encoder_cpu.py pins it to the stored outputs of the unmodified reference."""
from __future__ import annotations

import torch
import torch.nn.functional as F


@torch.no_grad()
def encoder_forward(enc, input_values: torch.Tensor, seq_len: int, output_hidden_states: bool = True):
    """-> (last_hidden_state [B, seq_len, H], tuple of hidden_states or None), fp32, on the module's device."""
    feats = enc.feature_extractor(input_values).transpose(1, 2)                          # [B, T6, 512]
    feats = F.interpolate(feats.transpose(1, 2), size=int(seq_len), align_corners=True, mode="linear").transpose(1, 2)
    hidden, _ = enc.feature_projection(feats)
    out = enc.encoder(hidden, attention_mask=None, output_attentions=False, output_hidden_states=output_hidden_states,
                      return_dict=True)
    return out.last_hidden_state, out.hidden_states


@torch.no_grad()
def mesh_infer(model, input_values: torch.Tensor, seq_len: int) -> torch.Tensor:
    """Audio2MeshModel.infer: out_fn(in_fn(features)), features = last hidden state or the mean of all hidden states."""
    last, states = encoder_forward(model.audio_encoder, input_values, seq_len, output_hidden_states=True)
    feats = last if model._only_last_features else sum(states) / len(states)
    return model.out_fn(model.in_fn(feats))


# ----------------------------------------------------------------------------------------------------------------------
# seeded weights and inputs of the audio goldens (tests/golden/audio_encoder_reference_s*.pt, oracle/make_golden_audio.py)
# ----------------------------------------------------------------------------------------------------------------------
A2M_SEED, A2P_SEED, INPUT_SEED, ID_SEED = 501, 502, 503, 7
SAMPLES = (21920, 80000, 85920)     # odd frame counts at conv layers 0, 2, 4, 5 / the 5 s pose chunk / the merged last chunk


def seq_len_of(samples: int) -> int:
    """scripts/audio2vid.py's frame count at 30 fps for a 16 kHz clip: ceil(S / 16000 * 30)."""
    import math
    return int(math.ceil(samples / 16000 * 30))


def waveform(samples: int, seed: int = INPUT_SEED) -> torch.Tensor:
    """Seeded waveform [1, S], normalised to zero mean and unit variance (what Wav2Vec2FeatureExtractor feeds the model)."""
    g = torch.Generator().manual_seed(seed * 1000003 + samples)
    x = torch.randn(1, samples, generator=g) * torch.linspace(0.2, 1.0, samples) + 0.1
    return (x - x.mean()) / torch.sqrt(x.var(unbiased=False) + 1e-7)


def seeded_state_dict(sd: dict, seed: int) -> dict:
    """randomize_state_dict(seed), then every wav2vec2 LayerNorm / GroupNorm scale and the positional convolution's
    weight-norm magnitude set to 1 + 0.1 randn (randomize_state_dict's name rules leave those near zero)."""
    import zlib
    from aniportrait_b200.synthetic import randomize_state_dict
    out = randomize_state_dict(sd, seed=seed)
    for name, t in out.items():
        if "audio_encoder." not in name:
            continue
        if name.endswith("layer_norm.weight") or name.endswith("weight.original0") or name.endswith("weight_g"):
            g = torch.Generator().manual_seed((seed * 7919 + zlib.crc32(name.encode())) & 0x7FFFFFFF)
            out[name] = (1.0 + 0.1 * torch.randn(t.shape, generator=g)).to(t.dtype)
    return out


def state_checksums(sd: dict) -> dict:
    """Per-tensor {shape, sum, sum of squares} in float64: a key-name or initialisation drift shows up here, not as a
    parity failure."""
    return {k: (tuple(v.shape), float(v.double().sum()), float(v.double().square().sum()))
            for k, v in sd.items() if v.is_floating_point()}
