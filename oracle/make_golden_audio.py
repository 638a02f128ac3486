"""TEST INFRASTRUCTURE — generates tests/golden/audio_encoder_reference_s{21920,80000,85920}.pt by running the UNMODIFIED
reference Audio2MeshModel.infer (src/audio_models/model.py:58-69) and Audio2PoseModel.infer (pose_model.py:97-124) on CPU
in fp32, with the full wav2vec2-base configuration (transformers' Wav2Vec2Config defaults) and the seeded weights and
waveforms of oracle/audio.py.

    ANIPORTRAIT_REFERENCE=<checkout> python oracle/make_golden_audio.py

Stored per waveform length: last_hidden_state and the Audio2Mesh output (fp32 for the 21920-sample case, which also pins
oracle/audio.py on the CPU; fp16 for the two long cases, compared on the GPU only), per-tensor checksums of the state dicts
the tests re-create, and for the short case the Audio2Pose output with the crops of its positional table and ALiBi mask.
Every file stays under 1 MB.
"""
from __future__ import annotations

import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import audio as OA  # noqa: E402
from oracle import ref_import  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def main():
    ref_import.activate()
    from transformers import Wav2Vec2Config
    from src.audio_models.model import Audio2MeshModel
    from src.audio_models.pose_model import Audio2PoseModel
    t0 = time.time()
    with tempfile.TemporaryDirectory() as cfg_dir:
        cfg = Wav2Vec2Config()
        cfg._attn_implementation = "eager"        # the reference's wrapper asks for attention maps
        cfg.save_pretrained(cfg_dir)
        a2m = Audio2MeshModel(dict(out_dim=1404, latent_dim=512, model_path=cfg_dir, only_last_fetures=True,
                                   from_pretrained=False)).eval()
        a2p = Audio2PoseModel(dict(out_dim=6, latent_dim=512, model_path=cfg_dir, only_last_fetures=True,
                                   from_pretrained=False)).eval()
    for m in (a2m, a2p):
        m.audio_encoder.config._attn_implementation = "eager"
    sd_m = OA.seeded_state_dict(a2m.state_dict(), OA.A2M_SEED)
    a2m.load_state_dict(sd_m)
    sd_p = OA.seeded_state_dict(a2p.state_dict(), OA.A2P_SEED)
    a2p.load_state_dict(sd_p)
    sums_m = OA.state_checksums(a2m.state_dict())
    sums_p = OA.state_checksums({k: v for k, v in a2p.state_dict().items() if k != "PPE.pe"})
    for S in OA.SAMPLES:
        T = OA.seq_len_of(S)
        x = OA.waveform(S)
        with torch.no_grad():
            emb = a2m.audio_encoder(x, seq_len=T, output_hidden_states=True)
            mesh = a2m.infer(x, T)
        short = S == OA.SAMPLES[0]
        dt = torch.float32 if short else torch.float16
        out = dict(samples=S, seq_len=T, waveform_sum=float(x.double().sum()), waveform_sq=float(x.double().square().sum()),
                   last_hidden_state=emb.last_hidden_state.to(dt).contiguous(), mesh=mesh.to(dt).contiguous(),
                   a2m_checksums=sums_m, torch_version=str(torch.__version__),
                   generator="reference src/audio_models model.py Audio2MeshModel / pose_model.py Audio2PoseModel, fp32 CPU")
        if short:
            with torch.no_grad():
                pose = a2p.infer(x, T, id_seed=torch.tensor([OA.ID_SEED]))
                pose_feats = a2p.audio_encoder(x, seq_len=T, output_hidden_states=True).last_hidden_state
            out.update(pose=pose.contiguous(), pose_features=pose_feats.contiguous(), a2p_checksums=sums_p,
                       pe=a2p.PPE.pe[:, :T].clone(), biased_mask=a2p.biased_mask[:, :T, :T].clone())
        path = os.path.join(GOLDEN, f"audio_encoder_reference_s{S}.pt")
        torch.save(out, path)
        print(f"{os.path.basename(path)}: seq_len {T}, {os.path.getsize(path) / 1e6:.2f} MB")
    print(f"audio_encoder_reference: {time.time() - t0:.1f}s")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count() or 8)
    main()
