"""Stand-ins for the reference's Audio2MeshModel / Audio2PoseModel (src/audio_models/model.py, pose_model.py) built from
transformers' Wav2Vec2Model and torch modules, with the reference's attribute and state-dict names, loaded with the seeded
weights of oracle/audio.py. The goldens of tests/golden/audio_encoder_reference_s*.pt were made with the real classes;
the per-tensor checksums stored there show that these stand-ins hold the same parameters."""
import os

import torch
from torch import nn

from oracle import audio as OA

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def golden(samples):
    return torch.load(os.path.join(ROOT, "tests", "golden", f"audio_encoder_reference_s{samples}.pt"))


def wav2vec2_base(**overrides):
    from transformers import Wav2Vec2Config, Wav2Vec2Model
    return Wav2Vec2Model(Wav2Vec2Config(**overrides))


class Audio2MeshStandIn(nn.Module):
    def __init__(self, encoder, latent_dim=512, out_dim=1404, only_last=True):
        super().__init__()
        self._only_last_features = only_last
        self.audio_encoder = encoder
        self.in_fn = nn.Linear(encoder.config.hidden_size, latent_dim)
        self.out_fn = nn.Linear(latent_dim, out_dim)

    def infer(self, input_value, seq_len):
        return OA.mesh_infer(self, input_value, seq_len)


class Audio2PoseStandIn(nn.Module):
    def __init__(self, encoder, pe, biased_mask, latent_dim=512, out_dim=6):
        super().__init__()
        self.out_dim = out_dim
        self._only_last_features = True
        self.audio_encoder = encoder
        self.pose_map = nn.Linear(out_dim, latent_dim)
        self.in_fn = nn.Linear(encoder.config.hidden_size, latent_dim)
        self.PPE = nn.Module()
        self.PPE.register_buffer("pe", pe)
        self.biased_mask = biased_mask
        layer = nn.TransformerDecoderLayer(d_model=latent_dim, nhead=8, dim_feedforward=2 * latent_dim, batch_first=True)
        self.transformer_decoder = nn.TransformerDecoder(layer, num_layers=8)
        self.pose_map_r = nn.Linear(latent_dim, out_dim)
        self.id_embed = nn.Embedding(100, latent_dim)


def build_a2m():
    m = Audio2MeshStandIn(wav2vec2_base())
    m.load_state_dict(OA.seeded_state_dict(m.state_dict(), OA.A2M_SEED))
    return m.eval()


def build_a2p(gold):
    m = Audio2PoseStandIn(wav2vec2_base(), gold["pe"], gold["biased_mask"])
    sd = {k: v for k, v in m.state_dict().items() if k != "PPE.pe"}
    m.load_state_dict(OA.seeded_state_dict(sd, OA.A2P_SEED), strict=False)
    return m.eval()


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm()).item()
