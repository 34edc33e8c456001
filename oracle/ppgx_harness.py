"""Reference import harness for the PPG extractor (TEST INFRASTRUCTURE - never imported by the product path), on top of
``ref_harness``: the extra stand-ins ``models/ppg_extractor`` needs to import and run on the CPU.  Like ``ref_harness`` it
exists only where the reference tree does; nothing under ``tests -m gpu``, ``bench*.py`` or ``smoke()`` imports it."""
from __future__ import annotations

import sys
import types

from ref_harness import REFERENCE_ROOT, install, reference_available  # noqa: F401


def install_ppg_extractor() -> None:
    """Make ``import models.ppg_extractor`` work on the unmodified reference (idempotent).  It imports three things this
    environment does not have:
      * ``torch_complex.tensor.ComplexTensor`` (frontend.py:10): a minimal stand-in with ``.real``, ``.imag``, ``.dim()``,
        all the frontend uses on the inference path;
      * ``espnet.nets.pytorch_backend.transformer.embedding.PositionalEncoding`` (encoder/subsampling.py:4, only as the
        fallback when no pos_enc is passed): aliased to the reference's own encoder/embedding.py, loaded by path because
        importing it as a package runs the failing package ``__init__``;
      * ``librosa.filters.mel`` (log_mel.py:47): routed to the restatement with the current meaning of ``norm=1``
        (per-filter L1; ``norm="slaney"`` is the pre-0.8 area normalisation), transposed back to librosa's [n_mels, F]."""
    install()
    import importlib.util

    if "torch_complex.tensor" not in sys.modules:
        tc, tct = types.ModuleType("torch_complex"), types.ModuleType("torch_complex.tensor")

        class ComplexTensor:
            def __init__(self, real, imag):
                self.real, self.imag = real, imag

            def dim(self):
                return self.real.dim()

        tct.ComplexTensor = ComplexTensor
        tc.tensor = tct
        sys.modules["torch_complex"], sys.modules["torch_complex.tensor"] = tc, tct
    name = "espnet.nets.pytorch_backend.transformer.embedding"
    if name not in sys.modules:
        parts = name.split(".")
        for i in range(1, len(parts)):
            sys.modules.setdefault(".".join(parts[:i]), types.ModuleType(".".join(parts[:i])))
        spec = importlib.util.spec_from_file_location(
            "_ppgx_ref_embedding", REFERENCE_ROOT / "models" / "ppg_extractor" / "encoder" / "embedding.py")
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        sys.modules[name] = mod
    from mockingbird_b200.synthesizer.audio_host import ppg_melmat

    def mel(sr, n_fft, n_mels=128, fmin=0.0, fmax=None, htk=False, norm=1, **_):
        if htk:
            raise NotImplementedError("htk mel scale is not restated")
        return ppg_melmat(sr, n_fft, n_mels, fmin or 0.0, fmax if fmax is not None else sr / 2.0, norm=norm).T

    sys.modules["librosa"].filters.mel = mel


def build_ppg_extractor(args: dict, seed: int = 0):
    """Reference PPGModel as models/ppg_extractor/__init__.py:66-72 builds it (CPU, eval)."""
    install_ppg_extractor()
    import argparse

    import torch
    import models.ppg_extractor as E

    torch.manual_seed(seed)
    return E.build_model(argparse.Namespace(**args)).eval()
