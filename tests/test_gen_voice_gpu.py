"""Text to speech through mockingbird_b200.gen_voice with stand-in seeded weights: every document of ``synthesize_wavs`` is
bitwise its own ``synthesize_wav`` whatever else is in the call, and bitwise gen_one_wav's body (gen_voice.py:15-42) written
out with the package's single calls; ``main`` writes one 16-bit WAV per document under gen_voice's names."""
import json

import numpy as np
import pytest
import torch

import harvest_oracle as ho
import ref_init as ri
from mockingbird_b200 import gen_voice, run
from mockingbird_b200.encoder import inference as enc
from mockingbird_b200.synthesizer.inference import Synthesizer
from mockingbird_b200.vocoder.fregan import inference as fre
from mockingbird_b200.vocoder.hifigan import inference as voc

pytestmark = pytest.mark.gpu

SR = 16000
SYLLABLES = ["ni3", "hao3", "wo3", "men5", "zhong1", "guo2", "ren2", "shi4", "jie4", "da4", "jia1", "xie4", "peng2", "you3"]


def _pcm(x):
    return np.clip(np.rint(x * 32767.0), -32768, 32767).astype(np.int16)


def _sentence(rng):
    return " ".join(rng.choice(SYLLABLES, int(rng.integers(1, 12))))


def _documents(n, seed, max_sentences=30):
    rng = np.random.default_rng(seed)
    return [[_sentence(rng) for _ in range(int(rng.integers(1, max_sentences + 1)))] for _ in range(n)]


@pytest.fixture(scope="module")
def models():
    from mockingbird_b200.encoder.model import SpeakerEncoder

    saved = (enc._model, enc._device, voc.generator, voc._device, voc.output_sample_rate, fre.generator, fre._device,
             fre.output_sample_rate)
    syn = Synthesizer("unused.pt", verbose=False)
    syn.load_state(ri.tacotron_state_dict(0, r=2, randomize_bn=True))
    syn._model.seed = 77
    m = SpeakerEncoder()
    m.load_state_dict(ri.encoder_state_dict(0))
    enc.set_model(m)
    voc.load_state(ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_16K, 0), ri.HIFIGAN_CONFIG_16K, precision="f16x3")
    yield syn
    (enc._model, enc._device, voc.generator, voc._device, voc.output_sample_rate, fre.generator, fre._device,
     fre.output_sample_rate) = saved


@pytest.fixture(scope="module")
def ref_wav(tmp_path_factory):
    from scipy.io import wavfile

    p = tmp_path_factory.mktemp("tts_ref") / "ref_spk.wav"
    wavfile.write(str(p), 22050, _pcm(ho.speechlike(31, 4 * 22050, 22050)))
    return str(p)


def _embed(ref_wav):
    return enc.embed_utterances(Synthesizer.load_preprocess_wavs([ref_wav]))[0]


def _gen_one_wav(syn, embed, texts, seed, vocoder=voc, trim_silences=True):
    """gen_voice.py:15-42 with the package's single calls: each sentence from its own row seed (the many-text call on one
    text), host concatenation, the B = 1 vocoder call and gen_voice's numpy lines verbatim"""
    specs = []
    for j, t in enumerate(texts):
        specs += syn.synthesize_spectrograms_many([t], [embed], style_idx=-1, min_stop_token=4, steps=400,
                                                  seeds=[(seed + j) % (1 << 64)])
    breaks = [spec.shape[1] for spec in specs]
    spec = np.concatenate(specs, axis=1)
    if spec.shape[1]:
        generated_wav, output_sample_rate = vocoder.infer_waveform(spec)
    else:  # every sentence trimmed to nothing: no samples to vocode
        generated_wav = np.zeros(0, np.float32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        b_ends = np.cumsum(np.array(breaks) * syn.hparams.hop_size)
        b_starts = np.concatenate(([0], b_ends[:-1]))
        wavs = [generated_wav[start:end] for start, end, in zip(b_starts, b_ends)]
        breaks = [np.zeros(int(0.15 * syn.sample_rate))] * len(breaks)
        generated_wav = np.concatenate([i for w, b in zip(wavs, breaks) for i in (w, b)])
        if trim_silences:
            generated_wav = enc.preprocess_wav(generated_wav)
        generated_wav = generated_wav / np.abs(generated_wav).max() * 0.97
    return generated_wav


def _same(a, b, what):
    assert a.dtype == np.float64 and b.dtype == np.float64 and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    assert np.array_equal(a, b, equal_nan=True), what


def test_one_document_is_synthesize_spectrograms_many(models, ref_wav):
    syn = models
    doc = _documents(1, 1, 8)[0]
    wav, sr = gen_voice.synthesize_wav(syn, doc, ref_wav)
    assert sr == SR and wav.dtype == np.float64
    embed = _embed(ref_wav)
    # the default seed is the model's: sentence j draws from seed + j, as synthesize_spectrograms_many's default does
    specs = syn.synthesize_spectrograms_many(doc, [embed] * len(doc), style_idx=-1, min_stop_token=4, steps=400)
    one = [syn.synthesize_spectrograms_many([t], [embed], style_idx=-1, min_stop_token=4, steps=400, seeds=[77 + j])[0]
           for j, t in enumerate(doc)]
    assert all(np.array_equal(a, b) for a, b in zip(specs, one))
    _same(wav, _gen_one_wav(syn, embed, doc, 77), "one document")


def test_device_mels_are_the_host_mels(models, ref_wav):
    syn = models
    texts = [s for d in _documents(6, 2, 10) for s in d]
    embed = _embed(ref_wav)
    seeds = list(range(100, 100 + len(texts)))
    dev = syn.synthesize_spectrograms_device(texts, [embed] * len(texts), style_idx=-1, min_stop_token=4, steps=400,
                                             seeds=seeds)
    host = syn.synthesize_spectrograms_many(texts, [embed] * len(texts), style_idx=-1, min_stop_token=4, steps=400,
                                            seeds=seeds)
    for i, (d, h) in enumerate(zip(dev, host)):
        assert d.is_cuda and d.shape == h.shape and np.array_equal(d.cpu().numpy(), h), i


@pytest.mark.parametrize("n_docs", [1, 5, 40])
def test_many_documents(models, ref_wav, n_docs, monkeypatch):
    syn = models
    docs = _documents(n_docs, 10 + n_docs)
    if n_docs == 40:
        # one document of over two minutes, and a budget that splits the vocoder's batches around it
        rng = np.random.default_rng(3)
        docs[7] = [" ".join(rng.choice(SYLLABLES, 11)) for _ in range(500)]
        monkeypatch.setattr(gen_voice, "VOCODER_WORKSPACE_BUDGET", 256 << 20)
    seeds = [int(s) for s in np.random.default_rng(n_docs).integers(0, 1 << 63, n_docs)]
    seeds[0] = (1 << 64) - 3  # row seeds wrap around 2**64
    wavs, sr = gen_voice.synthesize_wavs(syn, docs, ref_wav, seeds=seeds)
    assert sr == SR and len(wavs) == n_docs
    embed = _embed(ref_wav)
    for d in range(n_docs):
        _same(wavs[d], _gen_one_wav(syn, embed, docs[d], seeds[d]), f"document {d} against gen_one_wav")
    if n_docs == 40:
        assert len(wavs[7]) > 120 * SR
        # the document's vocoded samples (its length less the breaks; the cuts only shorten it) exceed the cap's
        cap = voc.generator.frame_cap(256 << 20)
        assert cap * voc.generator.hop < len(wavs[7]) - len(docs[7]) * int(0.15 * SR), cap
    if n_docs >= 5:
        for d in (0, 1, n_docs - 1):
            one, _ = gen_voice.synthesize_wav(syn, docs[d], ref_wav, seed=seeds[d])
            _same(wavs[d], one, f"document {d} against its synthesize_wav")
        perm = np.random.default_rng(1).permutation(n_docs).tolist()
        got, _ = gen_voice.synthesize_wavs(syn, [docs[i] for i in perm], ref_wav, seeds=[seeds[i] for i in perm])
        for k, i in enumerate(perm):
            _same(got[k], wavs[i], f"document {i} permuted")
        sub = [3, 1, 3, 3]  # a sub-list with duplicates
        got, _ = gen_voice.synthesize_wavs(syn, [docs[i] for i in sub], ref_wav, seeds=[seeds[i] for i in sub])
        for k, i in enumerate(sub):
            _same(got[k], wavs[i], f"document {i} in a sub-list")


@pytest.mark.parametrize("precision", ["f16tc"])
def test_vocoder_precisions(models, ref_wav, precision):
    syn = models
    saved = voc.generator, voc.output_sample_rate
    voc.load_state(ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_16K, 0), ri.HIFIGAN_CONFIG_16K, precision=precision)
    try:
        docs = _documents(4, 20, 12)
        wavs, _ = gen_voice.synthesize_wavs(syn, docs, ref_wav, seeds=[1, 2, 3, 4])
        embed = _embed(ref_wav)
        for d in range(4):
            _same(wavs[d], _gen_one_wav(syn, embed, docs[d], d + 1), f"{precision} document {d}")
    finally:
        voc.generator, voc.output_sample_rate = saved


def test_fregan_and_no_trim(models, ref_wav):
    syn = models
    fre.load_state(ri.fregan_state_dict(ri.FREGAN_CONFIG, 0), ri.FREGAN_CONFIG, precision="f16x3")
    docs = _documents(3, 30, 9)
    embed = _embed(ref_wav)
    wavs, _ = gen_voice.synthesize_wavs(syn, docs, ref_wav, seeds=[5, 6, 7], vocoder=fre)
    for d in range(3):
        _same(wavs[d], _gen_one_wav(syn, embed, docs[d], d + 5, vocoder=fre), f"fre-gan document {d}")
    wavs, _ = gen_voice.synthesize_wavs(syn, docs, ref_wav, seeds=[5, 6, 7], trim_silences=False)
    for d in range(3):
        _same(wavs[d], _gen_one_wav(syn, embed, docs[d], d + 5, trim_silences=False), f"untrimmed document {d}")
        assert np.abs(wavs[d]).max() == 0.97 or np.isnan(wavs[d]).all()


def test_timeline(models, ref_wav):
    timeline = []
    gen_voice.synthesize_wavs(models, _documents(2, 40, 4), ref_wav, timeline=timeline)
    torch.cuda.synchronize()
    stages = [s for s, _ in timeline[1:]]
    assert stages == ["reference", "tacotron", "join_mels", "vocoder", "breaks_levelling", "to_host"]
    assert all(timeline[0].elapsed_time(ev) >= 0 for _, ev in timeline[1:])


def test_main_writes_gen_voice_s_files(models, ref_wav, tmp_path, monkeypatch):
    from scipy.io import wavfile

    (tmp_path / "enc").mkdir()
    (tmp_path / "syn").mkdir()
    (tmp_path / "voc").mkdir()
    torch.save({"model_state": ri.encoder_state_dict(0), "step": 1}, tmp_path / "enc" / "pretrained.pt")
    sd = ri.tacotron_state_dict(0, r=2, randomize_bn=True)
    sd["step"] = torch.tensor(5)
    torch.save({"model_state": sd}, tmp_path / "syn" / "mandarin.pt")
    torch.save({"generator": ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_16K, 0)}, tmp_path / "voc" / "g_hifigan.pt")
    (tmp_path / "voc" / "config.json").write_text(json.dumps(ri.HIFIGAN_CONFIG_16K))
    rng = np.random.default_rng(8)
    lines = []
    for _ in range(30):  # about three documents of 1500 characters
        lines.append("，".join(" ".join(rng.choice(SYLLABLES, 8)) for _ in range(6)))
    text_file = tmp_path / "story.txt"
    text_file.write_text("\n".join(lines) + "\n")
    monkeypatch.chdir(tmp_path)
    saved = enc._model, enc._device, voc.generator, voc._device, voc.output_sample_rate
    try:
        written = gen_voice.main(["story.txt", ref_wav, "--enc_model_fpath", str(tmp_path / "enc" / "pretrained.pt"),
                                  "--syn_model_fpath", str(tmp_path / "syn" / "mandarin.pt"),
                                  "--voc_model_fpath", str(tmp_path / "voc" / "g_hifigan.pt")])
        docs = gen_voice.split_documents("\n".join(lines) + "\n")
        assert len(docs) >= 2
        assert written == [f"story.txt_{k}_ref_spk.wav.wav" for k in range(1, len(docs) + 1)]
        assert sorted(p.name for p in tmp_path.glob("*.wav")) == sorted(written)
        syn = Synthesizer(tmp_path / "syn" / "mandarin.pt", verbose=False)
        wavs, sr = gen_voice.synthesize_wavs(syn, docs, ref_wav)
        for name, w in zip(written, wavs):
            run.write_pcm16(tmp_path / "want.wav", w, sr)
            rate, pcm = wavfile.read(str(tmp_path / name))
            assert rate == SR and pcm.dtype == np.int16
            assert np.array_equal(pcm, wavfile.read(str(tmp_path / "want.wav"))[1]), name
    finally:
        enc._model, enc._device, voc.generator, voc._device, voc.output_sample_rate = saved
