"""HiFi-GAN ``infer_waveforms`` on CUDA mels (vocoder/_gan.py): every waveform is bitwise the utterance's B = 1 forward and
the host-mel ``infer_waveforms`` result, for the 24 kHz and 16 kHz generators in every precision."""
import numpy as np
import pytest
import torch

import ref_init as ri
from mockingbird_b200.vocoder._gan import infer_waveforms_batched
from mockingbird_b200.vocoder.hifigan.models import Generator

pytestmark = pytest.mark.gpu

CONFIGS = {"24k": ri.HIFIGAN_CONFIG_24K, "16k": ri.HIFIGAN_CONFIG_16K}


@pytest.fixture(scope="module")
def sds():
    return {name: ri.hifigan_state_dict(cfg, 0) for name, cfg in CONFIGS.items()}


@pytest.mark.parametrize("precision", ["f16tc", "f16x3", "fp32"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_device_mels_equal_single_and_host_calls(sds, name, precision):
    g = Generator(CONFIGS[name], precision=precision).cuda()
    g.load_state_dict(sds[name])
    g.eval()
    g.remove_weight_norm()
    lens = [40, 17, 64, 1, 33, 64, 5]
    gen = torch.Generator().manual_seed(5)
    host = [(torch.rand(80, t, generator=gen) * 8 - 4).numpy() for t in lens]
    dev = [torch.from_numpy(m).cuda() for m in host]
    dev[4] = torch.from_numpy(np.ascontiguousarray(host[4].T)).cuda().t()  # a transposed view, as a decoder's mel is
    with torch.no_grad():
        got = infer_waveforms_batched(g, "cuda", dev, batch_size=3)
        from_host = infer_waveforms_batched(g, "cuda", host, batch_size=3)
        for i, t in enumerate(lens):
            assert got[i].is_cuda and got[i].shape == (t * g.hop,), i
            alone = g(dev[i][None].contiguous())[0, 0]
            assert torch.equal(got[i], alone), i
            assert np.array_equal(got[i].cpu().numpy(), from_host[i]), i


def test_module_infer_waveforms_and_mixed_lists(sds):
    from mockingbird_b200.vocoder.hifigan import inference as gan_vocoder

    saved = gan_vocoder.generator, gan_vocoder._device, gan_vocoder.output_sample_rate
    try:
        gan_vocoder.load_state(sds["24k"], ri.HIFIGAN_CONFIG_24K, precision="fp32")
        mels = [torch.rand(80, t, generator=torch.Generator().manual_seed(t)).cuda() * 8 - 4 for t in (9, 30, 2)]
        with torch.no_grad():
            wavs = gan_vocoder.infer_waveforms(mels)
            for m, w in zip(mels, wavs):
                assert torch.equal(w, gan_vocoder.generator(m[None])[0, 0])
        with pytest.raises(ValueError, match="all CUDA tensors or all host arrays"):
            gan_vocoder.infer_waveforms([mels[0], mels[1].cpu().numpy()])
        with pytest.raises(ValueError, match=r"must be \[80, T\]"):
            gan_vocoder.infer_waveforms([mels[0][:40]])
    finally:
        gan_vocoder.generator, gan_vocoder._device, gan_vocoder.output_sample_rate = saved
