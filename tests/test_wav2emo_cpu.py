"""The wav2vec2 emotion model without a GPU: the float64 restatement pinned to the goldens recorded from the live reference,
the feature extractor's normalisation, frame counts, the weight-norm fold, create-time refusals and create_emo's files."""
from __future__ import annotations

import ctypes as C
import json
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT / "synth_weights"))

import gan_oracle as go  # noqa: E402
import ref_init as ri  # noqa: E402
import wav2emo_oracle as wo  # noqa: E402
from mockingbird_b200 import _lib  # noqa: E402
from mockingbird_b200.synthesizer.models import wav2emo as we  # noqa: E402

Z = np.load(ROOT / "tests" / "golden" / "wav2emo_seed0.npz")
CASES = ["small", *ri.WAV2EMO_SMALL_VARIANTS]


def _cfg(name):
    return ri.WAV2EMO_CONFIG_SMALL if name == "small" else ri.wav2emo_variant(name)


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_variants(name):
    cfg = _cfg(name)
    r = wo.forward(ri.wav2emo_state_dict(cfg, 0), cfg, Z["v_norm"])
    assert r["last"].shape[0] == int(Z[f"v_{name}_frames"])
    for key in ("emb", "logits"):
        e = go.rel_errors(r[key], torch.from_numpy(Z[f"v_{name}_{key}"]))
        assert e["max_rel"] <= 1e-5 and e["rms_rel"] <= 1e-5, (key, e)


def test_oracle_matches_reference_standin():
    cfg = ri.WAV2EMO_CONFIG
    r = wo.forward(ri.wav2emo_state_dict(cfg, 0), cfg, Z["a_norm"])
    for got, ref in ((r["emb"], Z["a_emb"]), (r["logits"], Z["a_logits"]), (r["last"][[0, 7, -1]], Z["a_rows"])):
        e = go.rel_errors(got, torch.from_numpy(ref))
        assert e["max_rel"] <= 1e-5 and e["rms_rel"] <= 1e-5, e


@pytest.mark.parametrize("case", ["a", "b", "tiny"])
def test_normalisation_bitwise_feature_extractor(case):
    y = wo.normalize(Z[f"{case}_wav"])
    assert y.dtype == np.float32 and np.array_equal(y.view(np.int32), Z[f"{case}_norm"].view(np.int32))


def test_frame_counts():
    assert int(Z["a_frames"]) == 149 == wo.num_frames(ri.WAV2EMO_CONFIG, 48000)
    assert int(Z["tiny_frames"]) == wo.num_frames(ri.WAV2EMO_CONFIG_SMALL, 400)
    assert wo.num_frames(ri.WAV2EMO_CONFIG, 400) == 1 and wo.num_frames(ri.WAV2EMO_CONFIG, 399) == 0
    m = we.EmotionExtractorModel(ri.WAV2EMO_CONFIG)
    for n in (0, 399, 400, 401, 21920, 48000, 480000):
        assert m.num_frames(n) == wo.num_frames(ri.WAV2EMO_CONFIG, n), n


def test_weight_norm_spellings_fold_alike():
    cfg = ri.WAV2EMO_CONFIG_SMALL
    sd = ri.wav2emo_state_dict(cfg, 0)
    p = "wav2vec2.encoder.pos_conv_embed.conv."
    old = {k.replace("parametrizations.weight.original0", "weight_g").replace("parametrizations.weight.original1", "weight_v"): v
           for k, v in sd.items()}
    a, b = we.fold_pos_conv(sd), we.fold_pos_conv(old)
    assert set(a) == set(b) and p + "weight" in a and not any("original" in k or "weight_g" in k for k in a)
    assert torch.equal(a[p + "weight"], b[p + "weight"])
    ref = wo.pos_conv_weight(sd)
    assert torch.allclose(a[p + "weight"].double(), ref, rtol=1e-6, atol=1e-7)


def test_fold_weight_norm_default_dim_unchanged():
    from mockingbird_b200.vocoder._gan import fold_weight_norm

    g = torch.Generator().manual_seed(0)
    v = torch.randn(6, 4, 3, generator=g)
    gg = torch.rand(6, 1, 1, generator=g)
    w = fold_weight_norm({"c.weight_g": gg, "c.weight_v": v})["c.weight"]
    assert torch.equal(w, v * (gg / v.reshape(6, -1).norm(dim=1).reshape(-1, 1, 1)))


@pytest.mark.parametrize("change", [
    dict(feat_extract_norm="group"), dict(do_stable_layer_norm=False), dict(hidden_act="relu"),
    dict(feat_extract_activation="gelu_new"), dict(add_adapter=True), dict(hidden_size=128, num_attention_heads=4),
    dict(intermediate_size=200), dict(conv_dim=[96] * 5), dict(num_conv_pos_embedding_groups=4),
    dict(conv_kernel=[10, 3, 3, 2, 7]),
])
def test_create_refuses(change):
    with pytest.raises(_lib.MbError):
        we.EmotionExtractorModel(dict(ri.WAV2EMO_CONFIG_SMALL, **change))


def test_config_json_parsing(tmp_path):
    cfg = dict(ri.WAV2EMO_CONFIG, id2label={"0": "arousal", "1": "dominance", "2": "valence"})
    cfg.pop("num_labels")
    c = we.make_config(json.loads(json.dumps(cfg)))
    assert (c.hidden_size, c.num_hidden_layers, c.num_attention_heads, c.num_labels) == (1024, 12, 16, 3)
    assert list(c.conv_kernel)[:7] == [10, 3, 3, 3, 3, 2, 2] and c.num_conv_layers == 7 and c.conv_bias == 1
    assert (c.feat_extract_norm, c.do_stable_layer_norm, c.hidden_act) == (0, 1, 0)
    assert abs(c.layer_norm_eps - 1e-5) < 1e-12
    obj = SimpleNamespace(**ri.WAV2EMO_CONFIG_SMALL)
    assert we.make_config(obj).hidden_size == 128
    with pytest.raises(_lib.MbError, match="local directory"):
        we.EmotionExtractorModel.from_pretrained("audeering/wav2vec2-large-robust-12-ft-emotion-msp-dim")


def test_create_emo_files_and_skip_existing(tmp_path, monkeypatch):
    from mockingbird_b200.synthesizer import preprocess_audio as pa

    (tmp_path / "audio").mkdir()
    names = ["audio-a_00.npy", "audio-b_01.npy", "audio-c_02.npy"]
    for i, n in enumerate(names):
        np.save(tmp_path / "audio" / n, np.full(400 + i, 0.1, np.float32))
    (tmp_path / "train.txt").write_text("".join(f"{n}|mel-{n}|embed-{n}|1|2|text\n" for n in names), encoding="utf-8")
    calls = []

    def fake(wavs, sampling_rate, embeddings=True, as_tensor=False):
        calls.append([len(w) for w in wavs])
        return [np.full(8, len(w), np.float64) for w in wavs]

    monkeypatch.setattr(pa, "extract_emos", fake)
    hp = SimpleNamespace(sample_rate=16000)
    (tmp_path / "emo").mkdir()
    np.save(tmp_path / "emo" / "emo-b_01.npy", np.zeros(8, np.float32))
    written = pa.create_emo(tmp_path, True, hp, batch_clips=1)
    assert [p.name for p in written] == ["emo-a_00.npy", "emo-c_02.npy"] and calls == [[400], [402]]
    v = np.load(tmp_path / "emo" / "emo-c_02.npy")
    assert v.dtype == np.float32 and v.shape == (8,) and v[0] == 402
    assert np.load(tmp_path / "emo" / "emo-b_01.npy")[0] == 0
    written = pa.create_emo(tmp_path, False, hp, n_processes=4)
    assert len(written) == 3 and calls[-1] == [400, 401, 402]


def test_extract_emo_refuses_other_rates():
    from mockingbird_b200.synthesizer import preprocess_audio as pa

    with pytest.raises(ValueError, match="16000"):
        pa.extract_emo(np.zeros(16000, np.float32), 22050)
