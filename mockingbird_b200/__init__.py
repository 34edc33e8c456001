"""mockingbird_b200: H100-native (sm_90a) vocoder / mel-synthesizer inference hot path of
babysor/MockingBird behind the reference's own Python inference surfaces.

    from mockingbird_b200.vocoder.hifigan import inference as gan_vocoder
    from mockingbird_b200.vocoder.wavernn import inference as rnn_vocoder
    from mockingbird_b200.vocoder.fregan import inference as fgan_vocoder

The compute path is the CUDA library built from mockingbird_b200/csrc (see include/mockingbird_b200.h);
importing the package does not touch the GPU.
"""
__version__ = "0.1.0"
