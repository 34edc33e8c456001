"""Fre-GAN ``FreGAN`` generator on the H100 path (reference: models/vocoder/fregan/generator.py:79-179)."""
from __future__ import annotations

from ... import _lib
from .._gan import GanGenerator

# models/vocoder/fregan/config.json (the generator-relevant keys)
DEFAULT_CONFIG = {
    "resblock": "1",
    "seed": 1234,
    "upsample_rates": [5, 5, 2, 2, 2],
    "upsample_kernel_sizes": [10, 10, 4, 4, 4],
    "upsample_initial_channel": 512,
    "resblock_kernel_sizes": [3, 7, 11],
    "resblock_dilation_sizes": [[1, 3, 5, 7], [1, 3, 5, 7], [1, 3, 5, 7]],
    "num_mels": 80,
    "hop_size": 200,
    "sampling_rate": 16000,
}


class FreGAN(GanGenerator):
    """``FreGAN(h, top_k=4)``; ``forward(mel[B,80,T]) -> wav[B,1,200*T]`` (generator.py:137-166)."""

    KIND = _lib.MB_GAN_FREGAN

    def __init__(self, h, top_k: int = 4, precision: str = "auto"):
        super().__init__(h, precision=precision, top_k=top_k)
