"""The workspace contract of every handle's compute calls (include/mockingbird_b200.h, Conventions), through the public
host API with `_lib.workspace` replaced:
  - a workspace of exactly *_workspace_bytes that starts 16 bytes past a torch allocation gives bitwise the same output as
    the library's own (aligned) workspace;
  - a NULL workspace is MB_ERR_INVALID and one byte short is MB_ERR_WORKSPACE, and neither counts a launch."""
import numpy as np
import pytest
import torch

import ref_init as ri
from mockingbird_b200 import _lib

pytestmark = pytest.mark.gpu


class _Null:
    """a workspace at address 0 that claims `n` bytes"""

    def __init__(self, n, device):
        self.n, self.device = n, device

    def data_ptr(self):
        return 0

    def numel(self):
        return self.n


def _patched(monkeypatch, mode):
    """_lib.workspace handing out `mode` workspaces: 'offset' (exact size, 16 bytes past an allocation), 'short', 'null'"""
    touched = []

    def workspace(need, device, owner=None, attr="_ws"):
        if mode == "null":
            ws = _Null(need, device)
        else:
            n = need if mode == "offset" else need - 1
            ws = torch.empty(n + 16, dtype=torch.uint8, device=device)[16:]
            assert ws.numel() == n and ws.data_ptr() % 256 == 16
        if owner is not None:
            setattr(owner, attr, ws)
            touched.append((owner, attr))
        return ws

    monkeypatch.setattr(_lib, "workspace", workspace)
    return touched


def _unpatch(monkeypatch, touched):
    monkeypatch.undo()
    for owner, attr in touched:
        setattr(owner, attr, None)


def _flat(x):
    """every tensor / array in a (nested) result, on the host"""
    if isinstance(x, torch.Tensor):
        return [x.detach().cpu()]
    if isinstance(x, np.ndarray):
        return [torch.from_numpy(np.ascontiguousarray(x))]
    if isinstance(x, (list, tuple)):
        return [t for v in x for t in _flat(v)]
    if isinstance(x, dict):
        return [t for k in sorted(x) for t in _flat(x[k])]
    if hasattr(x, "__dict__"):
        return _flat(vars(x))
    return []


# ---- one closure per compute entry point; each builds its model once and runs a small seeded call ----------------------

def _encoder():
    from mockingbird_b200.encoder.model import SpeakerEncoder

    m = SpeakerEncoder()
    m.load_state_dict(ri.encoder_state_dict(0))
    m.eval()
    return m


def case_encoder_frames():
    m = _encoder()
    x = torch.rand(3, 40, 40, generator=torch.Generator().manual_seed(1))
    return lambda: m.forward(x)


def case_encoder_rows():
    m = _encoder()
    frames = torch.rand(90, 40, generator=torch.Generator().manual_seed(2)).to(m.resolved_device())
    return lambda: m.embed_rows(frames, [0, 30, 50], [30, 20, 40])


def _tacotron():
    from mockingbird_b200.synthesizer.inference import Synthesizer

    return Synthesizer("unused.pt", verbose=False).load_state(ri.tacotron_state_dict(0, r=2, randomize_bn=True))


def _texts(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    seqs = [torch.randint(2, 75, (n,), generator=g) for n in lengths]
    emb = torch.rand(len(lengths), 256, generator=g)
    return seqs, emb / emb.norm(dim=1, keepdim=True)


def case_tacotron_padded():
    m = _tacotron()
    seqs, emb = _texts([20, 20], 3)
    chars = torch.stack(seqs)

    def run():
        torch.manual_seed(0)
        return m.generate(chars, emb, steps=30, style_idx=-1, min_stop_token=5)
    return run


def case_tacotron_ragged():
    m = _tacotron()
    seqs, emb = _texts([9, 25, 14], 4)
    return lambda: m.generate_many(seqs, emb, steps=[20, 30, 24], seeds=[1, 2, 3], min_stop_token=10)


def _gan(precision):
    from mockingbird_b200.vocoder.hifigan.models import Generator

    g = Generator(ri.HIFIGAN_CONFIG_16K, precision=precision).cuda()
    g.load_state_dict(ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_16K, 0))
    g.eval()
    g.remove_weight_norm()
    mel = torch.rand(2, 80, 24, generator=torch.Generator().manual_seed(5)).cuda() * 2 - 1
    return lambda: g(mel)


def case_gan_fp32():
    return _gan("fp32")


def case_gan_f16tc():
    return _gan("f16tc")


def case_gan_f16x3():
    return _gan("f16x3")


def _wavernn(mode):
    from mockingbird_b200.vocoder.wavernn import hparams as hp
    from mockingbird_b200.vocoder.wavernn import inference as rnn_vocoder

    old = hp.voc_mode
    try:
        hp.voc_mode = mode
        m = rnn_vocoder.load_state(ri.wavernn_state_dict(0, randomize_bn=True, mode=mode))
    finally:
        hp.voc_mode = old
        rnn_vocoder._model = None
    return m


def _mels(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(1, 80, T, generator=g) * 2 - 1 for T in lengths]


def case_wavernn_raw():
    m = _wavernn("RAW")
    mel = _mels([5], 6)[0]
    noise = torch.empty(380, 3, 512).exponential_(1, generator=torch.Generator().manual_seed(7))
    return lambda: m.generate_indices(mel, True, 300, 40, None, noise=noise)


def case_wavernn_postprocess():
    m = _wavernn("RAW")
    mel = _mels([30], 8)[0]

    def run():
        torch.manual_seed(0)
        return m.generate(mel, True, 1000, 100, True)
    return run


def case_wavernn_many_raw():
    m = _wavernn("RAW")
    mels = _mels([30, 27], 9)
    return lambda: m.generate_many(mels, True, 1000, 100, True, seeds=[5, 6], progress_callback=lambda *a: None)


def case_wavernn_many_mol():
    m = _wavernn("MOL")
    mels = _mels([28, 30], 10)
    return lambda: m.generate_many(mels, True, 1000, 100, True, seeds=[5, 6], progress_callback=lambda *a: None)


def case_deepmind():
    from mockingbird_b200.vocoder.wavernn.models.deepmind_version import WaveRNN

    m = WaveRNN(896, 256).cuda()
    m.load_state_dict(ri.deepmind_state_dict(0))
    noise = torch.empty(600, 2, 256).exponential_(1, generator=torch.Generator().manual_seed(11))
    return lambda: m.generate(600, noise=noise)


def case_ppg2mel():
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2

    m = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).cuda()
    m.load_state_dict(ri.ppg2mel_state_dict(0))
    m.eval()
    g = torch.Generator().manual_seed(12)
    lengths = [24, 17]
    utts = [(torch.randn(T, 144, generator=g),
             torch.stack([torch.randn(T, generator=g), (torch.rand(T, generator=g) < 0.7).float()], 1)) for T in lengths]
    spk = torch.randn(len(lengths), 256, generator=g)
    masks = [(torch.rand(2 * (T // 4), 256, generator=g) < 0.5, torch.rand(2 * (T // 4), 128, generator=g) < 0.5)
             for T in lengths]
    return lambda: m.inference_batch(utts, spk, dropout_masks=masks)


def case_ppgx():
    from mockingbird_b200.ppg_extractor import build_model

    m = build_model(ri.PPGX_CONFIG)
    m.load_state_dict(ri.ppg_extractor_state_dict(ri.PPGX_CONFIG, 0))
    m = m.cuda().eval()
    w = torch.randn(2, 8000, generator=torch.Generator().manual_seed(13)) * 0.1
    return lambda: m(w, torch.LongTensor([8000, 6000]))


def case_melspec_ragged():
    from mockingbird_b200.encoder import audio

    g = np.random.default_rng(14)
    wavs = [g.standard_normal(n).astype(np.float32) * 0.1 for n in (4000, 6400)]
    return lambda: audio.mel_front().many_flat(wavs)


def case_griffinlim():
    import griffinlim_oracle as go
    from mockingbird_b200.griffinlim import GriffinLim
    from mockingbird_b200.synthesizer.hparams import hparams as hp

    gl = GriffinLim(go.inv_basis(hp), hp.n_fft, hp.hop_size, hp.win_size, power=hp.power,
                    preemphasis=hp.preemphasis if hp.preemphasize else 0.0, signal_normalization=hp.signal_normalization,
                    allow_clipping=hp.allow_clipping_in_normalization, symmetric=hp.symmetric_mels,
                    max_abs_value=hp.max_abs_value, min_level_db=hp.min_level_db, ref_level_db=hp.ref_level_db)
    g = np.random.default_rng(15)
    mels = [(g.random((hp.num_mels, T)) * 8 - 4).astype(np.float32) for T in (20, 31)]
    return lambda: gl(mels, 3, seeds=[1, 2])


def _noises():
    g = np.random.default_rng(16)
    return [(g.standard_normal(n) * 0.05).astype(np.float32) for n in (4000, 5200)]


def case_logmmse_profile():
    from mockingbird_b200 import logmmse

    noises = _noises()
    return lambda: [p.noise_mu2 for p in logmmse.profile_noise_many(noises, 16000)]


def case_logmmse_denoise():
    from mockingbird_b200 import logmmse

    noises = _noises()
    profs = logmmse.profile_noise_many(noises, 16000)
    clips = [n * 3 for n in noises]
    return lambda: logmmse.denoise_many(clips, profs, 0.15)


def case_resample_forward():
    from mockingbird_b200 import resample as rs

    g = np.random.default_rng(17)
    clips = [(g.standard_normal(n) * 0.1).astype(np.float32) for n in (3000, 4410)]
    return lambda: rs.resample_many(clips, [24000, 44100], 16000)


def case_resample_level():
    from mockingbird_b200 import resample as rs

    g = np.random.default_rng(18)
    clips = rs.resample_device([(g.standard_normal(n) * 0.1).astype(np.float32) for n in (3000, 4410)], [16000, 16000], 16000)
    return lambda: (rs.mean_squares(clips), rs.normalize_volume_device(clips, -20), rs.rescale_device(clips, 0.9))


CASES = sorted(name[5:] for name in globals() if name.startswith("case_"))
_built = {}


def _run_of(name):
    if name not in _built:
        _built[name] = globals()["case_" + name]()
    return _built[name]


@pytest.mark.parametrize("name", CASES)
def test_misaligned_workspace_is_bitwise_equal(monkeypatch, name):
    run = _run_of(name)
    ref = _flat(run())
    touched = _patched(monkeypatch, "offset")
    try:
        got = _flat(run())
    finally:
        _unpatch(monkeypatch, touched)
    assert ref and len(got) == len(ref)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), (name, i)


@pytest.mark.parametrize("name", CASES)
def test_null_and_short_workspace_refused(monkeypatch, name):
    run = _run_of(name)
    run()  # uploads and first-use packing happen outside the counted window
    torch.cuda.synchronize()
    L = _lib.lib()
    for mode, status in (("null", 1), ("short", 4)):
        touched = _patched(monkeypatch, mode)
        n0 = L.mb_launch_count()
        try:
            with pytest.raises(_lib.MbError, match=f"error {status}:"):
                run()
        finally:
            _unpatch(monkeypatch, touched)
        assert L.mb_launch_count() == n0, (name, mode)
