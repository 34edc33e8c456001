"""The wav2vec2 emotion model on the GPU against the goldens recorded from the live reference and the float64 restatement,
ragged batches bitwise their single calls, the normalisation bitwise numpy's, snapshots, refusals and the VITS hand-off."""
from __future__ import annotations

import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT / "synth_weights"))

import gan_oracle as go  # noqa: E402
import ref_init as ri  # noqa: E402
import wav2emo_oracle as wo  # noqa: E402

pytestmark = pytest.mark.gpu
Z = np.load(ROOT / "tests" / "golden" / "wav2emo_seed0.npz")
TOL = 1e-4
MB_ERR_INVALID, MB_ERR_WORKSPACE = 1, 4  # include/mockingbird_b200.h


def _model(cfg):
    from mockingbird_b200.synthesizer.models.wav2emo import EmotionExtractorModel

    m = EmotionExtractorModel(cfg)
    m.load_state_dict(ri.wav2emo_state_dict(cfg, 0))
    return m.cuda().eval()


@pytest.fixture(scope="module")
def full():
    return _model(ri.WAV2EMO_CONFIG)


def _close(got, ref, tol=TOL):
    e = go.rel_errors(torch.as_tensor(got).cpu(), torch.as_tensor(ref))
    print(f"rel_errors {tuple(torch.as_tensor(ref).shape)}: {e}")
    assert e["max_rel"] <= tol and e["rms_rel"] <= tol, e
    return e


@pytest.mark.parametrize("case", ["a", "b"])
def test_standin_goldens(full, case):
    emb, logits, nrm, hid = full.run_clips([Z[f"{case}_wav"]], normed=True, hidden=True)[0]
    assert np.array_equal(nrm.cpu().numpy().view(np.int32), Z[f"{case}_norm"].view(np.int32))
    assert hid.shape[0] == int(Z[f"{case}_frames"])
    _close(emb, Z[f"{case}_emb"])
    _close(logits, Z[f"{case}_logits"])
    if case == "a":
        _close(hid[[0, 7, -1]], Z["a_rows"])
        r = wo.forward(ri.wav2emo_state_dict(ri.WAV2EMO_CONFIG, 0), ri.WAV2EMO_CONFIG, Z["a_norm"])
        _close(emb, r["emb"])
        _close(logits, r["logits"])
        _close(hid, r["last"])


@pytest.mark.parametrize("name", ["small", *ri.WAV2EMO_SMALL_VARIANTS])
def test_variant_goldens(name):
    cfg = ri.WAV2EMO_CONFIG_SMALL if name == "small" else ri.wav2emo_variant(name)
    m = _model(cfg)
    emb, logits, hid = m.run_clips([Z["v_wav"]], hidden=True)[0]
    assert hid.shape[0] == int(Z[f"v_{name}_frames"])
    _close(emb, Z[f"v_{name}_emb"])
    _close(logits, Z[f"v_{name}_logits"])
    r = wo.forward(ri.wav2emo_state_dict(cfg, 0), cfg, Z["v_norm"])
    _close(hid, r["last"])
    if name == "small":
        _close(hid, Z["v_small_last"])
        emb, logits, _ = m.run_clips([Z["tiny_wav"]], hidden=True)[0]
        _close(emb, Z["tiny_emb"])
        _close(logits, Z["tiny_logits"])


def test_thirty_seconds_against_oracle(full):
    rng = np.random.default_rng(3)
    wav = (0.3 * np.sin(np.arange(480000) * 0.05) + 0.05 * rng.standard_normal(480000)).astype(np.float32)
    emb, logits, nrm, hid = full.run_clips([wav], normed=True, hidden=True)[0]
    assert hid.shape[0] == 1499
    assert np.array_equal(nrm.cpu().numpy().view(np.int32), wo.normalize(wav).view(np.int32))
    r = wo.forward(ri.wav2emo_state_dict(ri.WAV2EMO_CONFIG, 0), ri.WAV2EMO_CONFIG, wo.normalize(wav))
    _close(emb, r["emb"])
    _close(logits, r["logits"])
    _close(hid, r["last"])


def test_call_matches_reference_forward(full):
    emb, logits = full(torch.from_numpy(Z["a_norm"])[None])
    assert emb.shape == (1, 1024) and logits.shape == (1, 3)
    _close(emb[0], Z["a_emb"])
    _close(logits[0], Z["a_logits"])


@pytest.mark.parametrize("count", [1, 5, 64, 130])
def test_ragged_rows_bitwise_single_calls(full, count):
    from mockingbird_b200.synthesizer import preprocess_audio as pa

    pa.load_model(full)
    rng = np.random.default_rng(count)
    lens = rng.integers(400, 480000, size=count)
    lens[0] = 400
    if count > 1:
        lens[1] = 480000
    wavs = [(0.2 * rng.standard_normal(int(n))).astype(np.float32) for n in lens]
    many = pa.extract_emos(wavs, 16000, True)
    for i in range(count):
        one = pa.extract_emo(wavs[i], 16000, True)
        assert one.shape == (1, 1024) and one.dtype == np.float32
        assert np.array_equal(one[0].view(np.int32), many[i].view(np.int32)), i
    logits = pa.extract_emo(wavs[0], 16000)
    assert logits.shape == (1, 3)


def test_from_pretrained_both_formats(tmp_path, full):
    from safetensors.torch import save_file

    from mockingbird_b200.synthesizer.models.wav2emo import EmotionExtractorModel

    cfg = ri.WAV2EMO_CONFIG_SMALL
    sd = ri.wav2emo_state_dict(cfg, 0)
    ref = _model(cfg).run_clips([Z["v_wav"]])[0][0].cpu()
    for fmt in ("bin", "safetensors"):
        d = tmp_path / fmt
        d.mkdir()
        (d / "config.json").write_text(json.dumps(cfg))
        if fmt == "bin":
            old = {k.replace("parametrizations.weight.original0", "weight_g").replace("parametrizations.weight.original1",
                                                                                       "weight_v"): v for k, v in sd.items()}
            torch.save(old, d / "pytorch_model.bin")
        else:
            save_file({k: v.contiguous() for k, v in sd.items()}, str(d / "model.safetensors"))
        m = EmotionExtractorModel.from_pretrained(d).cuda()
        got = m.run_clips([Z["v_wav"]])[0][0].cpu()
        assert torch.equal(got, ref), fmt


def test_refusals(full):
    from mockingbird_b200 import _lib
    from mockingbird_b200.synthesizer import preprocess_audio as pa

    pa.load_model(full)
    with pytest.raises(ValueError):
        pa.extract_emo(np.zeros(399, np.float32), 16000)
    with pytest.raises(ValueError):
        pa.extract_emo(np.zeros(22050, np.float32), 22050)
    import ctypes as C

    Lb = _lib.lib()
    full._prepare()
    need = int(Lb.mb_emo_workspace_bytes(full._handle, 1, 16000))
    wav = torch.zeros(16000, device="cuda")
    emb = torch.empty(1, 1024, device="cuda")
    lg = torch.empty(1, 3, device="cuda")
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    ns = (C.c_int32 * 1)(16000)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    assert Lb.mb_emo_forward(full._handle, p(wav), ns, 1, 1, p(emb), p(lg), None, None, p(ws), need - 1, st) == MB_ERR_WORKSPACE
    assert Lb.mb_emo_forward(full._handle, p(wav), ns, 1, 1, p(emb), p(lg), None, None, None, need, st) == MB_ERR_INVALID


def test_emos_feed_vits_infer_many(full):
    from mockingbird_b200.synthesizer import preprocess_audio as pa
    from mockingbird_b200.synthesizer.models.vits import Vits

    pa.load_model(full)
    rng = np.random.default_rng(5)
    wavs = [(0.2 * rng.standard_normal(n)).astype(np.float32) for n in (16000, 9000)]
    emos = pa.extract_emos(wavs, as_tensor=True)
    assert emos.is_cuda and emos.shape == (2, 1024) and emos.dtype == torch.float32
    v = Vits(**ri.VITS_TOY)
    v.load_state_dict(ri.vits_state_dict(ri.VITS_TOY, 0))
    v.cuda().eval()
    v.remove_weight_norm()
    texts = [torch.tensor([1, 2, 3, 4, 5]), torch.tensor([3, 4, 5])]
    a = v.infer_many(texts, [0, 1], emos, [1, 2])
    b = v.infer_many(texts, [0, 1], torch.from_numpy(np.stack(pa.extract_emos(wavs))), [1, 2])
    for x, y in zip(a, b):
        assert torch.equal(torch.as_tensor(x).cpu(), torch.as_tensor(y).cpu())
