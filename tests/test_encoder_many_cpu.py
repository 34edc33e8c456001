"""embed_utterances' host side: the row plan of each utterance, the plan of library calls, and the refusal of malformed
waveforms before anything is queued (no GPU needed)."""
import numpy as np
import pytest

from mockingbird_b200.encoder import inference as enc
from mockingbird_b200.encoder.params_data import partials_n_frames

HOP = 160


def _lengths():
    # exact hop boundaries, a coverage-drop case, short and long utterances
    return [0, 1, 159, 160, 161, 12799, 12800, 12801, 25599, 25600, 25601, 26000, 28000, 31999, 32000, 48000, 48123,
            16000 * 7 + 37, 16000 * 30]


@pytest.mark.parametrize("kwargs", [{}, {"overlap": 0.25}, {"overlap": 0.0}, {"rate": 2.0}, {"rate": 1.3},
                                    {"min_pad_coverage": 0.3}, {"min_pad_coverage": 1.0}])
def test_row_plan_equals_partial_slices(kwargs):
    for n in _lengths():
        sig, wave_slices, starts, lens = enc.utterance_rows(n, True, **kwargs)
        ws, ms = enc.compute_partial_slices(n, **kwargs)
        assert wave_slices == ws
        assert starts == [s.start for s in ms] and lens == [s.stop - s.start for s in ms]
        assert all(v == partials_n_frames for v in lens)
        # embed_utterance pads the waveform to wave_slices[-1].stop when that is not shorter
        assert sig == (ws[-1].stop if ws[-1].stop >= n else n)
        # the mel of the (virtually) padded signal covers every row
        assert 1 + sig // HOP >= starts[-1] + lens[-1]


def test_coverage_drop_case_is_covered():
    """a length whose last window is dropped for low coverage, and one where it is kept"""
    dropped = [n for n in range(25600, 48000, 160) if len(enc.compute_partial_slices(n)[0]) <
               len(enc.compute_partial_slices(n, min_pad_coverage=0.01)[0])]
    assert dropped
    n = dropped[0]
    sig, ws, starts, _ = enc.utterance_rows(n)
    assert len(starts) == len(enc.compute_partial_slices(n)[1]) and sig == max(n, ws[-1].stop)


def test_row_plan_without_partials():
    for n in _lengths():
        assert enc.utterance_rows(n, False) == (n, None, [0], [1 + n // HOP])


def test_call_plan_covers_every_row_once():
    rng = np.random.default_rng(0)
    row_lens = [[160] * int(k) for k in rng.integers(1, 40, 300)] + [[int(t)] for t in rng.integers(1, 4000, 50)]
    for max_rows, max_frames in ((1024, 1024 * 160), (7, 5000), (1, 1)):
        calls = enc.many_plan(row_lens, max_rows, max_frames)
        seen = {}
        for call in calls:
            rows = sum(r1 - r0 for _, r0, r1 in call)
            T = max(max(row_lens[u][r0:r1]) for u, r0, r1 in call)
            assert rows <= max_rows and (rows == 1 or rows * T <= max_frames)
            for u, r0, r1 in call:
                assert 0 <= r0 < r1 <= len(row_lens[u])
                for r in range(r0, r1):
                    assert (u, r) not in seen
                    seen[(u, r)] = True
        assert len(seen) == sum(len(v) for v in row_lens)
        # longest rows first
        firsts = [max(row_lens[u]) for call in calls for u, _, _ in call]
        assert firsts == sorted(firsts, reverse=True)
    assert enc.many_plan([]) == []
    with pytest.raises(ValueError):
        enc.many_plan([[160]], 0)


def test_call_plan_order():
    assert enc.many_plan([[160], [160] * 3, [160], [160] * 3], 4, 10 ** 6) == [[(1, 0, 3), (3, 0, 1)], [(3, 1, 3), (0, 0, 1),
                                                                                                         (2, 0, 1)]]
    assert enc.many_plan([[50], [300], [120]], 8, 600) == [[(1, 0, 1), (2, 0, 1)], [(0, 0, 1)]]


class _Loaded:
    """stands for a loaded model: the checks below refuse the input before any model or device is touched"""


@pytest.mark.parametrize("bad,match", [([np.zeros(3000, np.float32), np.zeros((2, 3000), np.float32)], "wav 1 has shape"),
                                       ([np.zeros(3000, np.float32), np.zeros(0, np.float32)], "wav 1 is empty")])
def test_malformed_waveforms_are_refused(bad, match):
    from mockingbird_b200.encoder import audio
    from mockingbird_b200.synthesizer import audio as saudio
    from mockingbird_b200.synthesizer.hparams import hparams

    saved = enc._model
    enc._model = _Loaded()
    try:
        with pytest.raises(ValueError, match=match):
            enc.embed_utterances(bad)
        with pytest.raises(ValueError, match=match):
            enc.embed_utterances(bad, using_partials=False)
    finally:
        enc._model = saved
    with pytest.raises(ValueError, match=match):
        audio.wav_to_mel_spectrograms(bad)
    with pytest.raises(ValueError, match=match):
        saudio.melspectrograms(bad, hparams)


def test_short_signal_is_refused():
    from mockingbird_b200.encoder import audio
    from mockingbird_b200.synthesizer import audio as saudio
    from mockingbird_b200.synthesizer.hparams import hparams

    wavs = [np.zeros(3000, np.float32), np.zeros(3000, np.float32), np.zeros(200, np.float32)]
    with pytest.raises(ValueError, match="wav 2 has 200 samples; reflect padding"):
        audio.wav_to_mel_spectrograms(wavs)
    with pytest.raises(ValueError, match="wav 2 has 200 samples; reflect padding"):
        saudio.melspectrograms(wavs, hparams)
    saved = enc._model
    enc._model = _Loaded()
    try:
        with pytest.raises(ValueError, match="wav 2 has 200 samples; reflect padding"):
            enc.embed_utterances(wavs, using_partials=False)
    finally:
        enc._model = saved


def test_not_loaded_error():
    saved = enc._model
    enc._model = None
    try:
        with pytest.raises(Exception, match="Model was not loaded"):
            enc.embed_utterances([np.zeros(16000, np.float32)])
    finally:
        enc._model = saved


def test_full_call_workspace_is_the_stated_figure():
    """a call of MANY_ROWS rows of 160 frames needs ~1.2 GB of workspace (the figure beside MANY_ROWS / MANY_FRAMES)"""
    import ctypes as C

    from mockingbird_b200 import _lib
    from mockingbird_b200.encoder.params_model import model_embedding_size, model_hidden_size, model_num_layers

    cfg = _lib.EncoderConfig()
    cfg.mel_n_channels, cfg.hidden_size, cfg.num_layers, cfg.embedding_size = 40, model_hidden_size, model_num_layers, \
        model_embedding_size
    h = C.c_void_p()
    L = _lib.lib()
    _lib.check(L.mb_encoder_create(C.byref(cfg), C.byref(h)))
    try:
        rows = int(L.mb_encoder_rows_workspace_bytes(h, enc.MANY_ROWS, enc.MANY_FRAMES // enc.MANY_ROWS))
        assert 1.1e9 < rows < 1.3e9, rows
        assert int(L.mb_encoder_rows_workspace_bytes(h, 0, 160)) == 0
    finally:
        L.mb_encoder_destroy(h)
