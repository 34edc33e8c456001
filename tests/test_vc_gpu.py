"""Voice conversion through mockingbird_b200.run with stand-in seeded weights: every clip of ``convert_wavs`` is bitwise its
``convert_wav`` call and bitwise run.py's loop body written out with the package's single-clip calls, and ``convert(args)``
writes one 16-bit WAV per source under run.py's names."""
import json

import numpy as np
import pytest
import torch

import harvest_oracle as ho
import ref_init as ri
from mockingbird_b200 import f0_utils as fu
from mockingbird_b200 import run
from mockingbird_b200.encoder import inference as enc
from mockingbird_b200.synthesizer import audio_host
from mockingbird_b200.vocoder.hifigan import inference as voc

pytestmark = pytest.mark.gpu

SR = 16000


def _pcm(x):
    return np.clip(np.rint(x * 32767.0), -32768, 32767).astype(np.int16)


@pytest.fixture(scope="module")
def models():
    from mockingbird_b200.encoder.model import SpeakerEncoder
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2
    from mockingbird_b200.ppg_extractor import build_model

    saved = enc._model, enc._device, voc.generator, voc._device, voc.output_sample_rate
    ext = build_model(ri.PPGX_CONFIG)
    ext.load_state_dict(ri.ppg_extractor_state_dict(ri.PPGX_CONFIG, 0))
    ext.cuda().eval()
    conv = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).cuda()
    conv.load_state_dict(ri.ppg2mel_state_dict(0))
    conv.eval()
    conv.seed = 1234
    m = SpeakerEncoder()
    m.load_state_dict(ri.encoder_state_dict(0))
    enc.set_model(m)
    voc.load_state(ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_24K, 0), ri.HIFIGAN_CONFIG_24K, precision="f16x3")
    yield ext, conv
    enc._model, enc._device, voc.generator, voc._device, voc.output_sample_rate = saved


@pytest.fixture(scope="module")
def clips(tmp_path_factory):
    """12 speech-like clips of 1-10 s: WAV paths at 16, 44.1 and 48 kHz and float32 arrays at 16 kHz; a 4 s reference WAV"""
    from scipy.io import wavfile

    d = tmp_path_factory.mktemp("vc_src")
    rng = np.random.default_rng(4)
    rates = [16000, 44100, 48000, None] * 3
    out = []
    for i, (sec, sr) in enumerate(zip(rng.uniform(1, 10, 12), rates)):
        rate = sr or SR
        x = ho.speechlike(200 + i, int(sec * rate), rate)
        if sr is None:
            out.append(x.astype(np.float32))
        else:
            p = d / f"src_{i:02d}.wav"
            wavfile.write(str(p), rate, _pcm(x))
            out.append(str(p))
    ref = d / "ref_spk.wav"
    wavfile.write(str(ref), SR, _pcm(ho.speechlike(99, 4 * SR)))
    return out, str(ref)


def test_many_equal_single(models, clips):
    ext, conv = models
    srcs, ref = clips
    seeds = [7 * i + 1 for i in range(len(srcs))]
    seeds[3] = (1 << 64) - 1
    many, sr = run.convert_wavs(ext, conv, srcs, ref, seeds=seeds)
    assert sr == 24000 and len(many) == len(srcs)
    for i, (src, s) in enumerate(zip(srcs, seeds)):
        one, sr1 = run.convert_wav(ext, conv, src, ref, seed=s)
        assert sr1 == 24000 and one.dtype == np.float32
        assert np.array_equal(many[i], one), i
    # reversed order and a sub-list give the same clips
    back, _ = run.convert_wavs(ext, conv, srcs[::-1], ref, seeds=seeds[::-1])
    assert all(np.array_equal(a, b) for a, b in zip(back[::-1], many))


def _run_py_loop(ext, conv, src, ref_path, seed):
    """run.py:51-91 for one source, with the package's single-clip calls (the speaker embedding by the many-clip call on
    one clip: the single-utterance embed_utterance is equal only to FP32 rounding)"""
    ref_wav = enc.preprocess_wav(ref_path)
    spk = torch.from_numpy(enc.embed_utterances([ref_wav])[0]).unsqueeze(0).cuda()
    ref_m, ref_s = fu.compute_mean_std(fu.f02lf0(fu.compute_f0(ref_wav)))
    src_wav = audio_host.load_wav(src, SR)[0] if isinstance(src, str) else src  # librosa.load(src_wav_path, sr=16000)
    ppg = ext.extract_from_wav(src_wav)
    lf0_uv = fu.get_converted_lf0uv(src_wav, ref_m, ref_s, convert=True)
    n = min(ppg.shape[1], len(lf0_uv))
    _, mel_pred, _ = conv.inference(ppg[:, :n], logf0_uv=torch.from_numpy(lf0_uv[:n]).unsqueeze(0).float().cuda(),
                                    spembs=spk, seed=seed)
    y, sr_out = voc.infer_waveform(mel_pred.transpose(0, 1).cpu())
    return y, sr_out


def test_equal_run_py_stage_by_stage(models, clips):
    ext, conv = models
    srcs, ref = clips
    many, _ = run.convert_wavs(ext, conv, srcs, ref)  # seeds=None: the convertor's seed for every clip
    for i, src in enumerate(srcs):
        y, sr = _run_py_loop(ext, conv, src, ref, conv.seed)
        assert sr == 24000
        assert np.array_equal(many[i], y), i


def test_convert_writes_run_py_outputs(models, clips, tmp_path):
    import yaml
    from scipy.io import wavfile

    srcs, ref = clips
    wav_dir = tmp_path / "wavs"
    wav_dir.mkdir()
    paths = [s for s in srcs if isinstance(s, str)][:4]
    for p in paths:
        (wav_dir / p.split("/")[-1]).write_bytes(open(p, "rb").read())
    (tmp_path / "ext").mkdir()
    sd = ri.ppg_extractor_state_dict(ri.PPGX_CONFIG, 0)
    torch.save({k: v for k, v in sd.items() if k.startswith("encoder.")}, tmp_path / "ext" / "24epoch.pt")
    (tmp_path / "ext" / "cfg.yaml").write_text(yaml.safe_dump(ri.PPGX_CONFIG))
    (tmp_path / "p2m").mkdir()
    (tmp_path / "p2m" / "train.yaml").write_text(yaml.safe_dump({"model": dict(ri.PPG2MEL_CONFIG)}))
    torch.save({"model": ri.ppg2mel_state_dict(0)}, tmp_path / "p2m" / "best_loss_step_000042.pth")
    (tmp_path / "voc").mkdir()
    torch.save({"generator": ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_24K, 0)}, tmp_path / "voc" / "g_02830000.pt")
    (tmp_path / "voc" / "config.json").write_text(json.dumps(ri.HIFIGAN_CONFIG_24K))
    torch.save({"model_state": ri.encoder_state_dict(0), "step": 5805000}, tmp_path / "enc.pt")
    out = tmp_path / "out"
    args = run.get_parser().parse_args([
        "--wav_dir", str(wav_dir), "--ref_wav_path", ref, "-c", str(tmp_path / "p2m" / "train.yaml"),
        "-m", str(tmp_path / "p2m" / "best_loss_step_000042.pth"), "-o", str(out),
        "--ppg_model_file", str(tmp_path / "ext" / "24epoch.pt"), "--vocoder_model_file", str(tmp_path / "voc" / "g_02830000.pt"),
        "--encoder_model_file", str(tmp_path / "enc.pt")])
    run.convert(args)
    names = sorted(p.name for p in out.iterdir())
    want = sorted(f"vc_{p.split('/')[-1][:-4]}_ref_ref_spk_step000042.wav" for p in paths)
    assert names == want
    # the written clips are the 16-bit PCM of convert_wavs with the models convert loaded, in sorted source order
    from mockingbird_b200.ppg_extractor import load_model

    ext = load_model(tmp_path / "ext" / "24epoch.pt")
    conv = run._build_ppg2mel_model({"model": dict(ri.PPG2MEL_CONFIG)}, tmp_path / "p2m" / "best_loss_step_000042.pth", "cuda")
    srcs_sorted = sorted(str(wav_dir / p.split("/")[-1]) for p in paths)
    wavs, sr = run.convert_wavs(ext, conv, srcs_sorted, ref)
    for src, w in zip(srcs_sorted, wavs):
        name = out / f"vc_{src.split('/')[-1][:-4]}_ref_ref_spk_step000042.wav"
        rate, pcm = wavfile.read(str(name))
        assert rate == 24000 and pcm.dtype == np.int16 and len(pcm) == len(w)
        x = np.clip(w, -1.0, 1.0).astype(np.float32) * np.float32(32767.0)
        assert np.array_equal(pcm, np.rint(x).astype(np.int16))
