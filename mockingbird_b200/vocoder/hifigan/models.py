"""HiFi-GAN ``Generator`` on the H100 path (reference: models/vocoder/hifigan/models.py:96-162)."""
from __future__ import annotations

from ... import _lib
from .._gan import GanGenerator

LRELU_SLOPE = 0.1

# models/vocoder/hifigan/config_16k_.json (the generator-relevant keys)
DEFAULT_CONFIG_16K = {
    "resblock": "1",
    "seed": 1234,
    "upsample_rates": [5, 5, 4, 2],
    "upsample_kernel_sizes": [10, 10, 8, 4],
    "upsample_initial_channel": 512,
    "resblock_kernel_sizes": [3, 7, 11],
    "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
    "num_mels": 80,
    "hop_size": 200,
    "sampling_rate": 16000,
}


class Generator(GanGenerator):
    """``Generator(h)``; ``forward(mel[B,80,T]) -> wav[B,1,hop*T]`` (models.py:134-150), hop = prod(h.upsample_rates).

    Like the reference (models.py:107-123), ``h.sampling_rate == 24000`` selects nearest-upsample + Conv1d upsampling layers
    (checkpoint keys ``ups.{i}.1.*``, odd kernel sizes only), every other rate ConvTranspose1d layers.

    ``precision``: "auto" (default; picks "f16tc" when a load-time probe shows it within 5e-4 of "f16x3" for this
    checkpoint, else "f16x3"), "f16tc" (wgmma, fp16 operands / fp32 accumulate, 3-term split on the serial layers),
    "f16x3" (wgmma, 3-term fp16 split everywhere: FP32-equivalent) or "fp32" (FFMA everywhere, ~1e-6)."""

    KIND = _lib.MB_GAN_HIFIGAN
