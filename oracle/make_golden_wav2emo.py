"""Record tests/golden/wav2emo_seed0.npz from the LIVE reference emotion model (TEST INFRASTRUCTURE).

Run in the build container only (needs the reference tree and transformers):

    CUDA_VISIBLE_DEVICES="" python oracle/make_golden_wav2emo.py

The unmodified ``models.synthesizer.models.wav2emo.EmotionExtractorModel`` runs on the CPU (eval, no grad) with the
stand-in configs of ``ref_init`` and ``ref_init.wav2emo_state_dict`` loaded strictly, which proves the transformers-5 key
names.  Under transformers 5 the class's ``init_weights()`` needs ``all_tied_weights_keys``; the harness sets that class
attribute to ``{}`` here and never edits the reference file.  Inputs go through ``Wav2Vec2FeatureExtractor`` (the
processor's feature extractor, do_normalize=True) and then, as a [1, n] batch, through the model.  No weights are stored.

Cases (wavs from make_golden_ppgx.synthetic_wav):
  a        WAV2EMO_CONFIG, 3 s: emb, logits, normalised input, and rows 0 / 7 / T - 1 of the last hidden state
  b        WAV2EMO_CONFIG, 1.37 s
  v_<name> WAV2EMO_CONFIG_SMALL ("small", with its whole last hidden state) and each variant of
           ref_init.WAV2EMO_SMALL_VARIANTS on one 0.9 s wav
  tiny     WAV2EMO_CONFIG_SMALL, 400 samples: the shortest clip with a frame
"""
from __future__ import annotations

import os
import sys
from pathlib import Path

os.environ.setdefault("CUDA_VISIBLE_DEVICES", "")
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent / "synth_weights"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import ref_harness  # noqa: E402
import ref_init as ri  # noqa: E402
from make_golden import GOLDEN, meta  # noqa: E402
from make_golden_ppgx import synthetic_wav  # noqa: E402

ROWS_A = (0, 7, -1)


def build(cfg: dict, seed: int = 0):
    from transformers import Wav2Vec2Config

    from models.synthesizer.models.wav2emo import EmotionExtractorModel

    EmotionExtractorModel.all_tied_weights_keys = {}
    m = EmotionExtractorModel(Wav2Vec2Config(**cfg))
    m.load_state_dict(ri.wav2emo_state_dict(cfg, seed), strict=True)
    return m.eval()


def run(m, wav: np.ndarray):
    from transformers import Wav2Vec2FeatureExtractor

    fe = Wav2Vec2FeatureExtractor(feature_size=1, sampling_rate=16000, padding_value=0.0, do_normalize=True,
                                  return_attention_mask=False)
    y = fe(wav, sampling_rate=16000)["input_values"][0]
    with torch.no_grad():
        out = m.wav2vec2(torch.from_numpy(y).reshape(1, -1))
        emb, logits = m(torch.from_numpy(y).reshape(1, -1))
    return y, emb[0].numpy(), logits[0].numpy(), out[0][0].numpy()


def main() -> None:
    # transformers probes optional packages when first imported: load it before the harness stubs them
    import transformers.models.wav2vec2.feature_extraction_wav2vec2  # noqa: F401
    import transformers.models.wav2vec2.modeling_wav2vec2  # noqa: F401

    ref_harness.install()
    torch.manual_seed(0)
    out = {}
    m = build(ri.WAV2EMO_CONFIG)
    for case, n, seed in (("a", 48000, 11), ("b", 21920, 12)):
        wav = synthetic_wav(n, seed)
        y, emb, logits, last = run(m, wav)
        out[f"{case}_wav"], out[f"{case}_norm"], out[f"{case}_emb"], out[f"{case}_logits"] = wav, y, emb, logits
        out[f"{case}_frames"] = np.int32(last.shape[0])
        if case == "a":
            out["a_rows"] = np.stack([last[r] for r in ROWS_A]).astype(np.float32)
    v_wav = synthetic_wav(14400, 13)
    out["v_wav"] = v_wav
    for name in ("small", *ri.WAV2EMO_SMALL_VARIANTS):
        cfg = ri.WAV2EMO_CONFIG_SMALL if name == "small" else ri.wav2emo_variant(name)
        y, emb, logits, last = run(build(cfg), v_wav)
        out[f"v_{name}_emb"], out[f"v_{name}_logits"] = emb, logits
        out[f"v_{name}_frames"] = np.int32(last.shape[0])
        if name == "small":
            out["v_small_last"] = last.astype(np.float32)
    out["v_norm"] = y
    tiny = synthetic_wav(400, 14)
    y, emb, logits, last = run(build(ri.WAV2EMO_CONFIG_SMALL), tiny)
    out.update(tiny_wav=tiny, tiny_norm=y, tiny_emb=emb, tiny_logits=logits, tiny_frames=np.int32(last.shape[0]))
    out["meta"] = np.array(meta(script="make_golden_wav2emo.py", transformers=__import__("transformers").__version__))
    np.savez_compressed(GOLDEN / "wav2emo_seed0.npz", **out)
    print("wrote", GOLDEN / "wav2emo_seed0.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
