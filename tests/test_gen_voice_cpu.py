"""CPU tests of the text-to-speech entry point (mockingbird_b200.gen_voice): gen_voice.py's document split restated, the
argument refusals before anything reaches the device, the output names and command line, float64 16-bit PCM, the vocoder's
padded-frame cap, and the host side of the new entries (workspace sizes, the break plan's clamped cuts, refusals)."""
import ctypes as C
import re

import numpy as np
import pytest

import ref_init as ri
from mockingbird_b200 import _lib, gen_voice, run
from mockingbird_b200.encoder import inference as enc
from mockingbird_b200.vocoder import _gan
from mockingbird_b200.vocoder.fregan import inference as fre
from mockingbird_b200.vocoder.hifigan import inference as voc


def _gen_voice_loop(input_txt):
    """gen_voice.py:76-96 as written there, collecting the documents gen_one_wav would receive"""
    docs = []
    texts = input_txt.split("\n")
    each_num = 1500
    punctuation = '！，。、,'
    processed_texts = []
    cur_num = 0
    for text in texts:
        for processed_text in re.sub(r'[{}]+'.format(punctuation), '\n', text).split('\n'):
            if processed_text:
                processed_texts.append(processed_text.strip())
                cur_num += len(processed_text.strip())
        if cur_num > each_num:
            docs.append(processed_texts)
            processed_texts = []
            cur_num = 0
    if len(processed_texts) > 0:
        docs.append(processed_texts)
    return docs


def _long_text():
    rng = np.random.default_rng(3)
    syll = ["ni3", "hao3", "wo3", "men5", "zhong1", "guo2", "ren2", "shi4"]
    lines = []
    for i in range(40):
        words = [" ".join(rng.choice(syll, rng.integers(3, 12))) for _ in range(rng.integers(1, 6))]
        lines.append(rng.choice(["，", "。", ",", "、", "！", "，，。"]).join(words))
    return "\n".join(lines)


TEXTS = [
    "",
    "\n\n",
    "ni3 hao3，shi4 jie4。wo3 lai2 le5",
    "a,,b，，c。。、d！e",
    ",，。leading and trailing punctuation。，",
    "  ,   ，x  , y ",  # whitespace-only pieces are kept as ""
    "one\ntwo，three\n\nfour,",
    "x" * 1501,  # one line over 1500 characters: a document by itself
    "x" * 1500 + "\n" + "y" * 10,  # exactly 1500 is not over: both lines in one document
    ("a" * 700 + "，") * 3 + "\n" + "tail，end",  # a line that crosses 1500, then a remainder
    _long_text(),
]


@pytest.mark.parametrize("text", TEXTS)
def test_split_documents_is_gen_voice_s_loop(text):
    assert gen_voice.split_documents(text) == _gen_voice_loop(text)


def test_split_documents_cases():
    assert gen_voice.split_documents("") == []
    assert gen_voice.split_documents("  ,   ，x  , y ") == [["", "", "x", "y"]]
    docs = gen_voice.split_documents("x" * 1501 + "\nshort")
    assert docs == [["x" * 1501], ["short"]]
    assert gen_voice.split_documents("ab，cd\nef", each_num=3) == [["ab", "cd"], ["ef"]]
    assert len(gen_voice.split_documents(_long_text(), each_num=200)) > 3


@pytest.fixture
def globals_restored():
    saved = enc._model, voc.generator, fre.generator
    yield
    enc._model, voc.generator, fre.generator = saved


def test_synthesize_wavs_argument_errors(globals_restored):
    clip = np.zeros(16000, np.float32)
    doc = ["ni3 hao3"]
    with pytest.raises(ValueError, match="no documents"):
        gen_voice.synthesize_wavs(None, [], clip)
    with pytest.raises(ValueError, match="document 1 has no sentences"):
        gen_voice.synthesize_wavs(None, [doc, []], clip)
    with pytest.raises(ValueError, match="document 0 is a string"):
        gen_voice.synthesize_wavs(None, ["ni3 hao3"], clip)
    with pytest.raises(ValueError, match="1 seeds for 2 documents"):
        gen_voice.synthesize_wavs(None, [doc, doc], clip, seeds=[3])
    for bad in (-1, 1 << 64, 1.5, True, "7"):
        with pytest.raises(ValueError, match=r"seeds\[1\]"):
            gen_voice.synthesize_wavs(None, [doc, doc], clip, seeds=[0, bad])
    with pytest.raises(ValueError, match="the vocoder must be"):
        gen_voice.synthesize_wavs(None, [doc], clip, vocoder=run)
    enc._model, voc.generator, fre.generator = None, None, None
    with pytest.raises(Exception, match="Model was not loaded"):
        gen_voice.synthesize_wavs(None, [doc], clip)
    enc._model = object()
    with pytest.raises(Exception, match="Please load hifi-gan"):
        gen_voice.synthesize_wav(None, doc, clip)
    with pytest.raises(Exception, match="Please load fre-gan"):
        gen_voice.synthesize_wav(None, doc, clip, vocoder=fre)
    # the largest seed is accepted (the error is the next check's)
    with pytest.raises(Exception, match="Please load hifi-gan"):
        gen_voice.synthesize_wavs(None, [doc, doc], clip, seeds=[0, (1 << 64) - 1])


def test_output_names():
    assert gen_voice.output_name("texts/story.txt", 3, "refs/spk_a.wav") == "texts/story.txt_3_spk_a.wav.wav"  # basename keeps its extension
    assert gen_voice.output_name("t.txt", 1, "ref.wav") == "t.txt_1_ref.wav.wav"


def test_parser_defaults_are_gen_voice_s():
    args = gen_voice.get_parser().parse_args(["story.txt", "ref.wav"])
    assert args.text_file == "story.txt" and args.wav_file == "ref.wav"
    # the checkpoints gen_voice.py hard-codes (gen_voice.py:111-113)
    assert args.enc_model_fpath == "encoder/saved_models/pretrained.pt"
    assert args.syn_model_fpath == "synthesizer/saved_models/mandarin.pt"
    assert args.voc_model_fpath == "vocoder/saved_models/pretrained/g_hifigan.pt"
    args = gen_voice.get_parser().parse_args(["s.txt", "r.wav", "--voc_model_fpath", "v.pt", "--enc_model_fpath", "e.pt",
                                              "--syn_model_fpath", "m.pt"])
    assert (args.enc_model_fpath, args.syn_model_fpath, args.voc_model_fpath) == ("e.pt", "m.pt", "v.pt")
    for missing in ([], ["story.txt"]):
        with pytest.raises(SystemExit):
            gen_voice.get_parser().parse_args(missing)


def _read(path):
    from scipy.io import wavfile

    sr, y = wavfile.read(str(path))
    assert y.dtype == np.int16
    return sr, y


def test_write_pcm16_float64(tmp_path):
    x = np.array([0.0, 0.5, -0.5, 1.0, -1.0, 1.7, -3.0, 1e-300], np.float64)
    run.write_pcm16(tmp_path / "a.wav", x, 16000)
    sr, y = _read(tmp_path / "a.wav")
    assert sr == 16000 and y.tolist() == [0, 16384, -16384, 32767, -32767, 32767, -32767, 0]  # clipped to +-32767
    # exact ties after the float64 scale round to even
    ties = [t for t in ((k + 0.5) / 32767 for k in range(-40, 40)) if t * 32767.0 == np.floor(t * 32767.0) + 0.5]
    assert len(ties) > 10
    run.write_pcm16(tmp_path / "t.wav", np.array(ties), 16000)
    got = _read(tmp_path / "t.wav")[1].astype(np.int64)
    assert all(v % 2 == 0 for v in got) and np.array_equal(got, np.rint(np.array(ties) * 32767.0))
    # float64 input is scaled in float64, not rounded to float32 first
    z = np.random.default_rng(0).uniform(-1.2, 1.2, 20000)
    run.write_pcm16(tmp_path / "z.wav", z, 16000)
    got = _read(tmp_path / "z.wav")[1]
    assert np.array_equal(got, np.clip(np.rint(z * 32767.0), -32767, 32767).astype(np.int16))
    via32 = np.rint(np.clip(z.astype(np.float32), -1.0, 1.0) * np.float32(32767.0)).astype(np.int16)
    assert not np.array_equal(got, via32)


def test_write_pcm16_float32_unchanged(tmp_path):
    x = np.array([0.0, 0.5, -0.5, 1.0, -1.0, 1.7, -3.0, 1.5 / 32767, 2.5 / 32767], np.float32)
    run.write_pcm16(tmp_path / "a.wav", x, 24000)
    sr, y = _read(tmp_path / "a.wav")
    assert sr == 24000 and y.tolist() == [0, 16384, -16384, 32767, -32767, 32767, -32767, 2, 2]
    rng = np.random.default_rng(0)
    z = rng.uniform(-1.2, 1.2, 5000).astype(np.float32)
    run.write_pcm16(tmp_path / "z.wav", z, 16000)
    assert np.array_equal(_read(tmp_path / "z.wav")[1], np.rint(np.clip(z, -1.0, 1.0) * np.float32(32767.0)).astype(np.int16))


def test_batches_frame_cap():
    lengths = [500, 300, 300, 200, 100, 5000, 50]
    order = sorted(range(len(lengths)), key=lambda i: -lengths[i])
    # no cap: runs of batch_size, as before
    assert _gan._batches(lengths, order, 3, None) == [order[0:3], order[3:6], order[6:7]]
    got = _gan._batches(lengths, order, 32, 1000)
    assert got == [[5], [0, 1], [2, 3, 4], [6]]  # 5000 alone; 2 x 500; 3 x 300; the last would make 4 x 300
    for b in got:
        assert [i for i in b] == [i for i in order if i in b]
        assert len(b) == 1 or len(b) * lengths[b[0]] <= 1000
    assert sum(got, []) == order
    assert _gan._batches(lengths, order, 2, 10 ** 9) == [order[0:2], order[2:4], order[4:6], order[6:7]]


def test_frame_cap_keeps_the_workspace_under_the_budget():
    from mockingbird_b200.vocoder.hifigan.models import Generator

    L = _lib.lib()
    for precision in ("fp32", "f16tc"):
        g = Generator(ri.HIFIGAN_CONFIG_16K, precision=precision)
        for budget in (64 << 20, 1 << 30, 4 << 30):
            cap = g.frame_cap(budget)
            assert cap >= 1
            for B in (1, 2, 7, 32):
                T = cap // B
                if T:
                    assert L.mb_gan_workspace_bytes(g._handle, B, T) <= budget, (precision, budget, B)
            assert L.mb_gan_workspace_bytes(g._handle, 32, -(-(cap + 32) // 32)) > budget
        assert g.frame_cap(1) == 1


def _up(n):
    return (n + 255) // 256 * 256


def test_workspace_sizes():
    L = _lib.lib()
    for B in (1, 3, 64, 65, 128):
        assert L.mb_tacotron_trim_workspace_bytes(B) == _up(4 * B) + 256
    for n in (1, 7, 8, 1000):
        assert L.mb_tts_join_workspace_bytes(n) == _up(32 * n) + 256  # 32-byte pieces
    for f in (L.mb_tacotron_trim_workspace_bytes, L.mb_tts_join_workspace_bytes, L.mb_resample_level_workspace_bytes):
        assert f(0) == 0 and f(-1) == 0


def _plan(pieces):
    L = _lib.lib()
    n = len(pieces)
    table = (_lib.TtsPiece * n)(*[_lib.TtsPiece(src, ln, a, b, z, 0) for src, ln, a, b, z in pieces])
    off = (C.c_int64 * (n + 1))()
    _lib.check(L.mb_tts_join_plan(table, n, off))
    return list(off)


def test_join_plan_is_numpy_slicing():
    """the plan's offsets are the lengths of numpy's x[start:end] plus the zeros, cut points past the row's end clamped"""
    src = 0x10000  # never dereferenced
    rng = np.random.default_rng(1)
    for _ in range(20):
        hop_syn, hop_voc = 256, int(rng.choice([200, 256, 300]))
        frames = rng.integers(0, 40, rng.integers(1, 9))
        n_row = int(frames.sum()) * hop_voc
        ends = np.cumsum(frames * hop_syn)
        starts = np.concatenate(([0], ends[:-1]))
        x = np.zeros(n_row)
        want = [0]
        for a, b in zip(starts, ends):
            want.append(want[-1] + len(x[a:b]) + 2400)
        got = _plan([(src if n_row else None, n_row, int(a), int(b), 2400) for a, b in zip(starts, ends)])
        assert got == want
    assert _plan([(None, 0, 0, 0, 0)]) == [0, 0]
    assert _plan([(src, 10, 4, 100, 3), (src, 10, 100, 200, 0)]) == [0, 9, 9]


def test_new_entries_refuse_before_the_device():
    L = _lib.lib()
    dev = C.c_void_p(0x10000)  # never dereferenced
    n0 = L.mb_launch_count()
    rows = (C.c_int32 * 3)(4, 9, 2)
    assert L.mb_tacotron_trim_frames(dev, 3, 80, 8, rows, C.c_float(-3.4), dev, dev, 1 << 20, None) == 1
    assert b"row 1 has 9 frames of 8" in L.mb_last_error()
    assert L.mb_tacotron_trim_frames(dev, 3, 80, 9, rows, C.c_float(-3.4), dev, dev, 16, None) != 0
    assert b"workspace too small" in L.mb_last_error()
    bad = [(0x10000, 10, 5, 4, 0)]
    table = (_lib.TtsPiece * 1)(*[_lib.TtsPiece(*p, 0) for p in bad])
    off = (C.c_int64 * 2)()
    assert L.mb_tts_join_plan(table, 1, off) == 1 and b"piece 0" in L.mb_last_error()
    assert L.mb_tts_join(table, 1, dev, dev, 1 << 20, None) == 1
    table = (_lib.TtsPiece * 1)(_lib.TtsPiece(None, 10, 0, 4, 0, 0))
    assert L.mb_tts_join(table, 1, dev, dev, 1 << 20, None) == 1 and b"null source row" in L.mb_last_error()
    assert L.mb_tts_join(table, 0, dev, dev, 1 << 20, None) == 1
    ok = (_lib.TtsPiece * 1)(_lib.TtsPiece(0x10000, 10, 0, 4, 0, 0))
    assert L.mb_tts_join(ok, 1, dev, dev, 16, None) != 0 and b"workspace too small" in L.mb_last_error()
    assert L.mb_launch_count() == n0
