"""Reference import harness (TEST INFRASTRUCTURE - never imported by the product path).

Imports the UNMODIFIED babysor/MockingBird modules from /root/reference (read-only) so that
``oracle/make_golden.py`` can generate golden vectors and so that the restatements under
``oracle/`` can be pinned against the real thing.  /root/reference exists only in the build
container, never on the GPU box: nothing under ``tests -m gpu``, ``bench.py`` or
``__graft_entry__.smoke()`` may import this file.

What it does (SURVEY.md section 8c / appendix C):
  * registers permissive stub modules for optional deps the reference imports at module scope
    but never uses on the inference hot path (matplotlib, librosa, soundfile, imp, pypinyin,
    webrtcvad, unidecode, inflect),
  * restores ``np.cumproduct`` (removed in NumPy 2; used at
    models/vocoder/wavernn/models/fatchord_version.py:64),
  * hides CUDA (the reference picks its device from torch.cuda.is_available() at call time,
    fatchord_version.py:164-167).
"""
from __future__ import annotations

import os
import sys
import types
from pathlib import Path

REFERENCE_ROOT = Path(os.environ.get("MOCKINGBIRD_REFERENCE", "/root/reference"))


def reference_available() -> bool:
    try:
        return (REFERENCE_ROOT / "models" / "vocoder" / "hifigan" / "models.py").is_file()
    except OSError:  # a parent directory this user may not traverse: the reference is absent
        return False


class _Stub(types.ModuleType):
    """Module whose every attribute is another stub / a no-op callable."""

    def __getattr__(self, name):
        if name.startswith("__") and name.endswith("__"):
            raise AttributeError(name)
        child = _Stub(f"{self.__name__}.{name}")
        setattr(self, name, child)
        return child

    def __call__(self, *a, **k):
        return None


_STUBS = [
    "matplotlib", "matplotlib.pyplot", "matplotlib.pylab", "matplotlib.cm",
    "librosa", "librosa.filters", "librosa.display", "librosa.effects", "librosa.util",
    "soundfile", "imp", "pypinyin", "webrtcvad", "unidecode", "inflect", "visdom", "umap",
]

_installed = False


def install() -> None:
    """Make ``import models.vocoder...`` resolve to the reference tree (idempotent)."""
    global _installed
    if _installed:
        return
    if not reference_available():
        raise RuntimeError(f"reference tree not found at {REFERENCE_ROOT}")
    import numpy as np

    if not hasattr(np, "cumproduct"):
        np.cumproduct = np.cumprod  # fatchord_version.py:64
    for name in _STUBS:
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                mod = _Stub(name)
                sys.modules[name] = mod
                if "." in name:
                    parent, child = name.rsplit(".", 1)
                    setattr(sys.modules[parent], child, mod)
    # pypinyin stub: lazy_pinyin(s, **kw) -> [s]; Style.TONE3 any constant
    pp = sys.modules["pypinyin"]
    if isinstance(pp, _Stub):
        pp.lazy_pinyin = lambda s, **kw: [s]
        pp.Style = types.SimpleNamespace(TONE3=8)
    ud = sys.modules["unidecode"]
    if isinstance(ud, _Stub):
        ud.unidecode = lambda s: s
    if str(REFERENCE_ROOT) not in sys.path:
        sys.path.insert(0, str(REFERENCE_ROOT))
    _installed = True


def hide_cuda() -> None:
    """Force the reference onto its CPU branches even on a GPU host."""
    import torch

    torch.cuda.is_available = lambda: False  # type: ignore[assignment]


def hifigan_config(name: str = "config_16k_.json") -> dict:
    import json

    with open(REFERENCE_ROOT / "models" / "vocoder" / "hifigan" / name) as f:
        return json.load(f)


def fregan_config() -> dict:
    import json

    with open(REFERENCE_ROOT / "models" / "vocoder" / "fregan" / "config.json") as f:
        return json.load(f)


def build_hifigan(seed: int = 0, rescale: float | None = None):
    """Reference Generator, eval, weight-norm folded (hifigan/inference.py:47-53)."""
    install()
    import torch
    from utils.util import AttrDict
    from models.vocoder.hifigan.models import Generator

    torch.manual_seed(seed)
    g = Generator(AttrDict(hifigan_config()))
    g.eval()
    g.remove_weight_norm()
    if rescale is not None:
        _variance_preserving_rescale(g, rescale)
    return g


def build_fregan(seed: int = 0, rescale: float | None = None):
    install()
    import torch
    from utils.util import AttrDict
    from models.vocoder.fregan.generator import FreGAN

    torch.manual_seed(seed)
    g = FreGAN(AttrDict(fregan_config()))
    g.eval()
    g.remove_weight_norm()
    if rescale is not None:
        _variance_preserving_rescale(g, rescale)
    return g


def _variance_preserving_rescale(module, gain: float) -> None:
    """init_weights uses std=0.01 (utils/util.py:55-58) which makes activations vanish through
    the stack; for a second, harder parity case re-draw every conv weight with a fan-in scaled
    std so that activations stay O(1) like a trained model's."""
    import math
    import torch

    with torch.no_grad():
        for m in module.modules():
            if isinstance(m, (torch.nn.Conv1d, torch.nn.ConvTranspose1d)):
                w = m.weight
                if isinstance(m, torch.nn.ConvTranspose1d):
                    fan_in = w.shape[0] * w.shape[2] / m.stride[0]
                else:
                    fan_in = w.shape[1] * w.shape[2]
                w.normal_(0.0, gain / math.sqrt(fan_in))
                if m.bias is not None:
                    m.bias.normal_(0.0, 0.05)


def build_wavernn(seed: int = 0):
    """Reference fatchord WaveRNN as wavernn/inference.py:8-25 builds it."""
    install()
    import torch
    from models.vocoder.wavernn.models.fatchord_version import WaveRNN
    from models.vocoder.wavernn import hparams as hp

    torch.manual_seed(seed)
    m = WaveRNN(rnn_dims=hp.voc_rnn_dims, fc_dims=hp.voc_fc_dims, bits=hp.bits, pad=hp.voc_pad,
                upsample_factors=hp.voc_upsample_factors, feat_dims=hp.num_mels,
                compute_dims=hp.voc_compute_dims, res_out_dims=hp.voc_res_out_dims,
                res_blocks=hp.voc_res_blocks, hop_length=hp.hop_length,
                sample_rate=hp.sample_rate, mode=hp.voc_mode)
    m.eval()
    return m


def build_tacotron(seed: int = 0):
    """Reference Tacotron as synthesizer/inference.py:52-65 builds it."""
    install()
    import torch
    from models.synthesizer.hparams import hparams
    from models.synthesizer.models.tacotron import Tacotron
    from models.synthesizer.utils.symbols import symbols

    torch.manual_seed(seed)
    m = Tacotron(embed_dims=hparams.tts_embed_dims, num_chars=len(symbols), encoder_dims=hparams.tts_encoder_dims,
                 decoder_dims=hparams.tts_decoder_dims, n_mels=hparams.num_mels, fft_bins=hparams.num_mels,
                 postnet_dims=hparams.tts_postnet_dims, encoder_K=hparams.tts_encoder_K, lstm_dims=hparams.tts_lstm_dims,
                 postnet_K=hparams.tts_postnet_K, num_highways=hparams.tts_num_highways, dropout=hparams.tts_dropout,
                 stop_threshold=hparams.tts_stop_threshold, speaker_embedding_size=hparams.speaker_embedding_size)
    m.eval()
    return m


def build_encoder(seed: int = 0):
    """Reference SpeakerEncoder as encoder/inference.py:31-34 builds it (CPU)."""
    install()
    import torch
    from models.encoder.model import SpeakerEncoder

    torch.manual_seed(seed)
    m = SpeakerEncoder(torch.device("cpu"), torch.device("cpu"))
    m.eval()
    return m


def load_deepmind():
    """Import the UNMODIFIED models/vocoder/wavernn/models/deepmind_version.py.  As shipped it star-imports two modules
    that do not exist in the tree (`utils.display`, `utils.dsp`) for the names time / np / stream / combine_signal, and
    calls `.cuda()` unconditionally: provide those names through stub modules and make `.cuda()` a CPU no-op while the
    returned class is in use (harness only; the reference file itself is untouched)."""
    install()
    import time as _time

    import numpy as _np
    import torch

    disp = types.ModuleType("utils.display")
    disp.time, disp.np, disp.stream = _time, _np, (lambda *a, **k: None)
    dsp = types.ModuleType("utils.dsp")
    dsp.combine_signal = lambda coarse, fine: coarse * 256 + fine - 2 ** 15  # wavernn/audio.py:34-35
    dsp.np = _np
    sys.modules["utils.display"], sys.modules["utils.dsp"] = disp, dsp
    import utils as _u

    _u.display, _u.dsp = disp, dsp
    torch.Tensor.cuda = lambda self, *a, **k: self  # type: ignore[assignment]
    from models.vocoder.wavernn.models.deepmind_version import WaveRNN

    return WaveRNN
