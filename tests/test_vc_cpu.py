"""CPU tests of the voice-conversion entry point (mockingbird_b200.run) and of ppg2mel's per-row dropout seeds: argument
validation before anything reaches the device, the frame trim, run.py's command line and output names, and the workspace
layout that holds the seed table."""
import ctypes as C

import numpy as np
import pytest
import torch

import ref_init as ri
from mockingbird_b200 import _lib, run
from mockingbird_b200.encoder import inference as enc
from mockingbird_b200.ppg2mel import MelDecoderMOLv2, seed_table
from mockingbird_b200.vocoder.hifigan import inference as voc


def _utts(lengths):
    g = torch.Generator().manual_seed(0)
    return [(torch.randn(T, 144, generator=g), torch.randn(T, 2, generator=g)) for T in lengths]


@pytest.fixture
def model():
    return MelDecoderMOLv2(**ri.PPG2MEL_CONFIG)


def test_inference_batch_seeds_validation(model):
    utts, spk = _utts([40, 12, 20]), torch.zeros(3, 256)
    with pytest.raises(ValueError, match="seeds alone"):
        model.inference_batch(utts, spk, seed=1, seeds=[1, 2, 3])
    masks = [(np.ones((20, 256)), np.ones((20, 128)))] * 3
    with pytest.raises(ValueError, match="seeds alone"):
        model.inference_batch(utts, spk, dropout_masks=masks, seeds=[1, 2, 3])
    with pytest.raises(ValueError, match="2 seeds for 3 utterances"):
        model.inference_batch(utts, spk, seeds=[1, 2])
    for bad in (-1, 1 << 64, 1.5, True, "7"):
        with pytest.raises(ValueError, match=r"seeds\[1\]"):
            model.inference_batch(utts, spk, seeds=[0, bad, 2])


def test_seed_table_keeps_64_bits():
    top = (1 << 64) - 1
    t = seed_table([0, 5, 1 << 63, top], 4)
    assert t == [0, 5, -(1 << 63), -1]
    assert torch.tensor(t, dtype=torch.int64).numpy().view(np.uint64).tolist() == [0, 5, 1 << 63, top]
    assert seed_table([], 0) == []


def _layout_bytes(B, T, seeds=True):
    """ws_layout of csrc/ppg2mel.cu: regions rounded up to 256 bytes, then 256 bytes of alignment slack"""
    up = lambda n: (n + 255) // 256 * 256  # noqa: E731
    T1, T2 = T // 2, T // 4
    S = 2 * T2
    f = [8 * 128 + 8, B * 256, B * T * 256, B * T1 * 256, B * T2 * 256, B * T2 * 256, B * T2 * 256, 2 * B * 512, B * 512,
         2 * B * 512, B * 512, B * 256, B * 8, B * 80, B * 128, B * 256, B * 2 * S * 512, B * 2 * S * 512]
    total = sum(up(4 * n) for n in f) + (up(8 * B) if seeds else 0)
    return total + 256


@pytest.mark.parametrize("B,T", [(1, 4), (1, 100), (7, 333), (33, 1000), (128, 1001)])
def test_workspace_holds_the_seed_table(B, T):
    """mb_ppg2mel_workspace_bytes counts B uint64 seeds (one 256-byte-aligned region) on top of the other regions"""
    lib = _lib.lib()
    from test_ppg2mel_cpu import _cfg

    h = C.c_void_p()
    _lib.check(lib.mb_ppg2mel_create(C.byref(_cfg()), C.byref(h)))
    try:
        got = lib.mb_ppg2mel_workspace_bytes(h, B, T)
        assert got == _layout_bytes(B, T)
        assert got - _layout_bytes(B, T, seeds=False) == (8 * B + 255) // 256 * 256
        assert got % 256 == 0
    finally:
        lib.mb_ppg2mel_destroy(h)


def test_rows_entry_refuses_before_the_device():
    """a NULL seed table and an unfinalized handle are refused without queuing anything"""
    lib = _lib.lib()
    from test_ppg2mel_cpu import _cfg

    h = C.c_void_p()
    _lib.check(lib.mb_ppg2mel_create(C.byref(_cfg()), C.byref(h)))
    dev = C.c_void_p(0x10000)  # never dereferenced
    lens = (C.c_int32 * 2)(8, 8)
    steps = (C.c_int32 * 2)()
    try:
        n0 = lib.mb_launch_count()
        args = lambda seeds: (h, dev, dev, dev, lens, 2, 8, seeds, dev, dev, dev, None, steps, dev, 1 << 30, None)  # noqa: E731
        assert lib.mb_ppg2mel_inference_rows(*args(None)) == 1
        assert b"null seed table" in lib.mb_last_error()
        assert lib.mb_ppg2mel_inference_rows(*args(dev)) == 2  # MB_ERR_STATE: weights not finalized
        assert b"mb_ppg2mel_inference_rows" in lib.mb_last_error()
        assert lib.mb_launch_count() == n0
    finally:
        lib.mb_ppg2mel_destroy(h)


def test_trim_pair_takes_the_shorter():
    ppg = torch.zeros(103, 144)
    lf0 = np.zeros((101, 2), np.float32)
    p, l = run.trim_pair(ppg, lf0)
    assert p.shape == (101, 144) and l.shape == (101, 2)
    p, l = run.trim_pair(ppg[:99], lf0)
    assert p.shape == (99, 144) and l.shape == (99, 2)
    p, l = run.trim_pair(ppg[:101], lf0)
    assert p.shape[0] == l.shape[0] == 101


@pytest.fixture
def globals_restored():
    saved = enc._model, voc.generator, voc.output_sample_rate
    yield
    enc._model, voc.generator, voc.output_sample_rate = saved


def test_convert_wavs_argument_errors(globals_restored):
    clip = np.zeros(16000, np.float32)
    with pytest.raises(ValueError, match="no source clips"):
        run.convert_wavs(None, None, [], clip)
    with pytest.raises(ValueError, match="1 seeds for 2 source clips"):
        run.convert_wavs(None, None, [clip, clip], clip, seeds=[3])
    enc._model, voc.generator = None, None
    with pytest.raises(Exception, match="Model was not loaded"):
        run.convert_wavs(None, None, [clip], clip)
    enc._model = object()
    with pytest.raises(Exception, match="Please load hifi-gan"):
        run.convert_wav(None, None, clip, clip)
    voc.generator, voc.output_sample_rate = object(), 16000
    with pytest.raises(ValueError, match="24000 Hz HiFi-GAN; the loaded vocoder is 16000 Hz"):
        run.convert_wav(None, None, clip, clip)


def test_parser_defaults_are_run_py_s():
    args = run.get_parser().parse_args(["--wav_dir", "src", "--ref_wav_path", "ref.wav", "-c", "cfg.yaml", "-m", "m.pth"])
    assert args.wav_dir == "src" and args.ref_wav_path == "ref.wav"
    assert args.ppg2mel_model_train_config == "cfg.yaml" and args.ppg2mel_model_file == "m.pth"
    assert args.output_dir == "vc_gens_vctk_oneshot"  # run.py:127-132
    # the checkpoints run.py hard-codes (run.py:41, 48, 56)
    assert args.ppg_model_file == "./ppg_extractor/saved_models/24epoch.pt"
    assert args.vocoder_model_file == "./vocoder/saved_models/24k/g_02830000.pt"
    assert args.encoder_model_file == "encoder/saved_models/pretrained_bak_5805000.pt"
    for missing in (["--ref_wav_path", "r.wav", "-c", "c", "-m", "m"], ["--wav_dir", "s", "-c", "c", "-m", "m"],
                    ["--wav_dir", "s", "--ref_wav_path", "r.wav", "-m", "m"],
                    ["--wav_dir", "s", "--ref_wav_path", "r.wav", "-c", "c"]):
        with pytest.raises(SystemExit):
            run.get_parser().parse_args(missing)


def test_output_names():
    step = run.checkpoint_step("ppg2mel/saved_models/vc/best_loss_step_304000.pth")
    assert step == "304000"
    assert run.checkpoint_step("x/model.pth") == "model"
    assert (run.output_name("out", "data/src/p225_001.wav", "refs/spk_a.wav", step)
            == "out/vc_p225_001_ref_spk_a_step304000.wav")


def test_write_pcm16(tmp_path):
    from scipy.io import wavfile

    x = np.array([0.0, 0.5, -0.5, 1.0, -1.0, 1.7, -3.0, 1.5 / 32767, 2.5 / 32767], np.float32)
    run.write_pcm16(tmp_path / "a.wav", x, 24000)
    sr, y = wavfile.read(str(tmp_path / "a.wav"))
    assert sr == 24000 and y.dtype == np.int16
    assert y.tolist() == [0, 16384, -16384, 32767, -32767, 32767, -32767, 2, 2]
