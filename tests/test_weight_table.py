"""The weight protocol every model handle shares (include/mockingbird_b200.h, Conventions): set_weight checks its
arguments, the name and the exact reference shape before the call order, derived tensors are not settable, and
set_arena forgets every tensor set before.  The CPU tests make no CUDA call: no arena is ever attached there, so no
set_weight reaches a copy."""
import ctypes as C

import pytest
import torch

import ref_init as ri
from mockingbird_b200 import _lib

MB_OK, MB_ERR_INVALID, MB_ERR_STATE, MB_ERR_WORKSPACE = 0, 1, 2, 4


def _gan(kind, cfg, sd, precision):
    from mockingbird_b200.vocoder.fregan.models import FreGAN
    from mockingbird_b200.vocoder.hifigan.models import Generator

    return (FreGAN if kind == "fregan" else Generator)(cfg, precision=precision), sd


def _fatchord(_):
    from mockingbird_b200.vocoder.wavernn.models.fatchord_version import WaveRNN

    hp = ri.WAVERNN_HP
    keys = ("rnn_dims", "fc_dims", "bits", "pad", "upsample_factors", "feat_dims", "compute_dims", "res_out_dims",
            "res_blocks", "hop_length", "sample_rate")
    return WaveRNN(**{k: hp[k] for k in keys}), ri.wavernn_state_dict(0)


def _deepmind(_):
    from mockingbird_b200.vocoder.wavernn.models.deepmind_version import WaveRNN

    return WaveRNN(896, 256), ri.deepmind_state_dict(0)


def _tacotron(_):
    from mockingbird_b200.synthesizer.models.tacotron import Tacotron

    return Tacotron(512, 75, 256, 128, 80, 80, 512, 5, 1024, 5, 4, 0.5, -3.4, 256), ri.tacotron_state_dict(0)


def _encoder(_):
    from mockingbird_b200.encoder.model import SpeakerEncoder

    return SpeakerEncoder(), ri.encoder_state_dict(0)


def _ppg2mel(_):
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2

    return MelDecoderMOLv2(**ri.PPG2MEL_CONFIG), ri.ppg2mel_state_dict(0)


def _ppgx(_):
    from mockingbird_b200.ppg_extractor import build_model

    return build_model(ri.PPGX_CONFIG), ri.ppg_extractor_state_dict(ri.PPGX_CONFIG, 0)


# name -> (C prefix, arena alignment, factory(gan precision) -> (module, state dict), derived tensor name or None)
MODELS = {
    "hifigan16k": ("gan", 256, lambda p: _gan("hifigan", ri.HIFIGAN_CONFIG_16K,
                                              ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_16K, 0), p), None),
    "hifigan24k": ("gan", 256, lambda p: _gan("hifigan", ri.HIFIGAN_CONFIG_24K,
                                              ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_24K, 0), p), None),
    "fregan": ("gan", 256, lambda p: _gan("fregan", ri.FREGAN_CONFIG, ri.fregan_state_dict(ri.FREGAN_CONFIG, 0), p), None),
    "fatchord": ("wavernn", 256, _fatchord, None),
    "deepmind": ("deepmind", 256, _deepmind, None),
    "tacotron": ("tacotron", 256, _tacotron, "decoder.mel_proj.packed"),
    "encoder": ("encoder", 256, _encoder, "lstm.bias_sum_l0"),
    "ppg2mel": ("ppg2mel", 256, _ppg2mel, None),
    "ppgx": ("ppgx", 1024, _ppgx, None),
}


def _fn(prefix, op):
    return getattr(_lib.lib(), f"mb_{prefix}_{op}")


def _finalize(prefix, handle):
    fin = _fn(prefix, "finalize")
    return fin(handle) if prefix == "gan" else fin(handle, None)


def _set(prefix, handle, name, t, dims):
    arr = None if dims is None else (C.c_int64 * max(1, len(dims)))(*dims)
    ndim = t.dim() if dims is None else len(dims)
    return _fn(prefix, "set_weight")(handle, name.encode(), C.c_void_p(t.data_ptr()), arr, ndim, None)


@pytest.fixture(scope="module", params=list(MODELS))
def model(request):
    prefix, align, make, derived = MODELS[request.param]
    m, sd = make("fp32")
    m.load_state_dict(sd)
    return prefix, align, m, m.weights_for_upload(), derived


def test_every_upload_tensor_passes_name_and_shape(model):
    """before set_arena, each tensor the host module uploads gets past the name and shape checks to the call order"""
    prefix, _, m, weights, _ = model
    assert weights
    for name, t in weights.items():
        t = t.float().contiguous()
        assert _set(prefix, m._handle, name, t, list(t.shape)) == MB_ERR_STATE, (name, _lib.lib().mb_last_error())


def test_bad_name_shape_and_arguments_are_invalid(model):
    prefix, _, m, weights, derived = model
    name, t = next((k, v) for k, v in weights.items() if v.dim() >= 2 and v.shape[0] != v.shape[1])
    t = t.float().contiguous()
    shape = list(t.shape)
    bad = {
        "transposed": [shape[1], shape[0]] + shape[2:],
        "flattened": [t.numel()],
        "extra leading dim": [1] + shape,
    }
    for what, dims in bad.items():
        assert _set(prefix, m._handle, name, t, dims) == MB_ERR_INVALID, (what, name, dims)
    assert _set(prefix, m._handle, "no.such.weight", t, shape) == MB_ERR_INVALID
    assert _set(prefix, m._handle, name, t, None) == MB_ERR_INVALID  # dims = NULL with ndim > 0
    if derived is not None:
        assert _set(prefix, m._handle, derived, t, [t.numel()]) == MB_ERR_INVALID, derived
        assert b"unknown" in _lib.lib().mb_last_error()


def test_set_arena_refusals_and_finalize_without_weights(model):
    prefix, align, m, _, _ = model
    set_arena = _fn(prefix, "set_arena")
    nbytes = int(_fn(prefix, "arena_bytes")(m._handle))
    assert nbytes > 0
    base = 1 << 32  # never dereferenced: every call below is refused before the handle keeps it
    assert set_arena(m._handle, None, nbytes) == MB_ERR_INVALID
    assert set_arena(m._handle, C.c_void_p(base + align // 2), nbytes) == MB_ERR_INVALID
    assert set_arena(m._handle, C.c_void_p(base), nbytes - 1) == MB_ERR_WORKSPACE
    assert _finalize(prefix, m._handle) == MB_ERR_STATE


def _compute(prefix, h, p):
    """the model's compute entry point on dummy device pointers: it must refuse before reading any of them"""
    L = _lib.lib()
    big = 1 << 30
    if prefix == "gan":
        return L.mb_gan_forward(h, p, None, 1, 8, p, p, big, None)
    if prefix == "wavernn":
        return L.mb_wavernn_generate(h, (C.c_int32 * 1)(0), 1, 10, 0, 10, None, 0, p, p, big, None)
    if prefix == "deepmind":
        return L.mb_deepmind_generate(h, 10, 0, 10, None, 0, p, p, p, big, None)
    if prefix == "tacotron":
        return L.mb_tacotron_generate(h, p, p, 1, 4, 10, 2, 0, 5.0, None, None, 0, p, p, None, C.byref(C.c_int32()), p,
                                      big, None)
    if prefix == "encoder":
        return L.mb_encoder_embed_frames(h, p, 1, 10, p, p, big, None)
    if prefix == "ppg2mel":
        return L.mb_ppg2mel_inference(h, p, p, p, (C.c_int32 * 1)(8), 1, 8, None, None, 0, p, p, p, None,
                                      (C.c_int32 * 1)(), p, big, None)
    assert prefix == "ppgx"
    return L.mb_ppgx_forward(h, p, (C.c_int32 * 1)(16000), 1, 16000, 5000, p, p, None, p, big, None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(MODELS))
def test_set_arena_forgets_uploaded_weights(name):
    """upload through the host module (finalize succeeds), then point the handle at a second zeroed arena: finalize
    and the compute entry point refuse with MB_ERR_STATE and launch nothing"""
    prefix, align, make, _ = MODELS[name]
    dev = torch.device("cuda", torch.cuda.current_device())
    m, sd = make("f16x3")
    m.load_state_dict(sd)
    m.to(dev)
    m._upload()
    assert m._ready and m._arena is not None
    L = _lib.lib()
    nbytes = int(_fn(prefix, "arena_bytes")(m._handle))
    second = torch.zeros(nbytes + align, dtype=torch.uint8, device=dev)
    base = (second.data_ptr() + align - 1) // align * align
    _lib.check(_fn(prefix, "set_arena")(m._handle, C.c_void_p(base), nbytes))
    assert _finalize(prefix, m._handle) == MB_ERR_STATE
    launches = L.mb_launch_count()
    assert _compute(prefix, m._handle, C.c_void_p(base)) == MB_ERR_STATE
    assert b"finalized" in L.mb_last_error()
    assert L.mb_launch_count() == launches
    torch.cuda.synchronize()
