"""Seeded re-creation of the reference's random-init weights WITHOUT the reference tree.

Synthetic-weight helper, NOT part of the oracle and not part of the product: the reference ships no checkpoints, so
tests/, bench.py and smoke() need seeded random-init weights of the reference architectures (there is no network to
fetch real ones).  Lives outside oracle/ so that bench.py / smoke() visibly import nothing from oracle/ when they build
their inputs; contains no forward arithmetic.

The reference ships no checkpoints (SURVEY.md section 4), so every parity case uses the weights
``torch.manual_seed(seed); Model(...)`` would produce.  /root/reference does not exist on the GPU
box and 13 M parameters are too large to commit as fixtures, so this file restates the *order in
which the reference constructors consume the global torch RNG* (module construction order and the
``.apply(init_weights)`` passes) and rebuilds the tensors from plain ``torch.nn`` layers:

  HiFi-GAN  Generator.__init__   models/vocoder/hifigan/models.py:96-132
  Fre-GAN   FreGAN.__init__      models/vocoder/fregan/generator.py:79-135
  WaveRNN   WaveRNN.__init__     models/vocoder/wavernn/models/fatchord_version.py:88-116

tests/test_oracle_pinned.py checks (in the build container, where the reference can be imported)
that these dicts are bit-identical to the reference modules' state_dicts, and the committed golden
outputs under tests/golden/ pin them on the GPU box.

Note: ``init_weights`` (utils/util.py:55-58) runs ``m.weight.data.normal_(0, 0.01)`` on modules that
are already wrapped by the old ``torch.nn.utils.weight_norm``; there ``m.weight`` is the derived
attribute, not ``weight_v``, so the draw is consumed from the RNG but does not change the
effective weights - they keep Conv1d's default kaiming-uniform init.
"""
from __future__ import annotations

import math
from typing import Dict

import torch


def _fold(w: torch.Tensor) -> torch.Tensor:
    """what remove_weight_norm leaves behind: _weight_norm(v, g=||v||, dim=0)."""
    g = torch.norm_except_dim(w, 2, 0)
    return torch._weight_norm(w, g, 0)


def _burn_normal(shape) -> None:
    torch.empty(shape).normal_(0.0, 0.01)


def _put(sd, name, m) -> None:
    sd[name + ".weight"] = _fold(m.weight.detach())
    sd[name + ".bias"] = m.bias.detach().clone()


def _resblocks(sd, cfg, n_stages: int) -> None:
    C0 = cfg["upsample_initial_channel"]
    ks, ds = cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"]
    nk = len(ks)
    for i in range(n_stages):
        ch = C0 // (2 ** (i + 1))
        for j, (k, d) in enumerate(zip(ks, ds)):
            base = f"resblocks.{i * nk + j}"
            if str(cfg["resblock"]) == "1":
                for group in ("convs1", "convs2"):
                    mods = [torch.nn.Conv1d(ch, ch, k) for _ in d]
                    for m_i, m in enumerate(mods):
                        _put(sd, f"{base}.{group}.{m_i}", m)
                    for m in mods:
                        _burn_normal(m.weight.shape)
            else:
                mods = [torch.nn.Conv1d(ch, ch, k) for _ in d]
                for m_i, m in enumerate(mods):
                    _put(sd, f"{base}.convs.{m_i}", m)
                for m in mods:
                    _burn_normal(m.weight.shape)


def hifigan_state_dict(cfg: dict, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Folded (weight-norm removed) generator weights of ``torch.manual_seed(seed); Generator(h)``.  At
    ``sampling_rate == 24000`` each upsampling layer is ``Sequential(InterpolationBlock(u), Conv1d(k))`` (models.py:107-118):
    its conv is ``ups.{i}.1`` and consumes the RNG where the ConvTranspose1d would."""
    torch.manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    C0 = cfg["upsample_initial_channel"]
    _put(sd, "conv_pre", torch.nn.Conv1d(80, C0, 7))
    interp = cfg.get("sampling_rate") == 24000
    ups = []
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        if interp:
            m = torch.nn.Conv1d(C0 // (2 ** i), C0 // (2 ** (i + 1)), k)
            _put(sd, f"ups.{i}.1", m)
        else:
            m = torch.nn.ConvTranspose1d(C0 // (2 ** i), C0 // (2 ** (i + 1)), k, u)
            _put(sd, f"ups.{i}", m)
        ups.append(m)
    _resblocks(sd, cfg, len(ups))
    post = torch.nn.Conv1d(C0 // (2 ** len(ups)), 1, 7)
    _put(sd, "conv_post", post)
    for m in ups:
        _burn_normal(m.weight.shape)
    _burn_normal(post.weight.shape)
    return sd


def fregan_state_dict(cfg: dict, seed: int = 0, top_k: int = 4) -> Dict[str, torch.Tensor]:
    torch.manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    C0 = cfg["upsample_initial_channel"]
    rates, kernels = cfg["upsample_rates"], cfg["upsample_kernel_sizes"]
    n_up = len(rates)
    _put(sd, "conv_pre", torch.nn.Conv1d(80, C0, 7))
    ups, cond_up, res_out = [], [], []
    kr = 80
    for i, (u, k) in enumerate(zip(rates, kernels)):
        m = torch.nn.ConvTranspose1d(C0 // (2 ** i), C0 // (2 ** (i + 1)), k, u)
        ups.append(m)
        _put(sd, f"ups.{i}", m)
        if i > (n_up - top_k):
            r = torch.nn.Conv1d(C0 // (2 ** i), C0 // (2 ** (i + 1)), 1)
            _put(sd, f"res_output.{len(res_out)}.1", r)
            res_out.append(r)
        if i >= (n_up - top_k):
            c = torch.nn.ConvTranspose1d(kr, C0 // (2 ** i), kernels[i - 1], rates[i - 1])
            _put(sd, f"cond_up.{len(cond_up)}", c)
            cond_up.append(c)
            kr = C0 // (2 ** i)
    _resblocks(sd, cfg, n_up)
    post = torch.nn.Conv1d(C0 // (2 ** n_up), 1, 7)
    _put(sd, "conv_post", post)
    for m in ups:
        _burn_normal(m.weight.shape)
    _burn_normal(post.weight.shape)
    for m in cond_up:
        _burn_normal(m.weight.shape)
    for m in res_out:
        _burn_normal(m.weight.shape)
    return sd


HIFIGAN_CONFIG_16K = {
    "resblock": "1", "seed": 1234,
    "upsample_rates": [5, 5, 4, 2], "upsample_kernel_sizes": [10, 10, 8, 4],
    "upsample_initial_channel": 512, "resblock_kernel_sizes": [3, 7, 11],
    "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
    "num_mels": 80, "hop_size": 200, "sampling_rate": 16000,
}

# 24 kHz HiFi-GAN (nearest upsample + Conv1d per stage, hop 240 = 10 ms frames).  A STAND-IN: the json of the released 24 kHz
# checkpoint (run.py:46, vocoder/saved_models/24k/) is not part of the reference tree, so these are plausible values with
# prod(upsample_rates) == hop_size and odd kernel sizes; the library itself takes every value from the caller's config.
HIFIGAN_CONFIG_24K = {
    "resblock": "1", "seed": 1234,
    "upsample_rates": [5, 4, 3, 2, 2], "upsample_kernel_sizes": [11, 9, 7, 5, 5],
    "upsample_initial_channel": 512, "resblock_kernel_sizes": [3, 7, 11],
    "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
    "num_mels": 80, "hop_size": 240, "sampling_rate": 24000,
}

# test-only second 24 kHz config: upsample rate 8, a kernel (17) wider than the tap conv's 11 taps before folding, ResBlock2
HIFIGAN_CONFIG_24K_U8 = {
    "resblock": "2", "seed": 1234,
    "upsample_rates": [8, 5, 3, 2], "upsample_kernel_sizes": [17, 11, 7, 5],
    "upsample_initial_channel": 256, "resblock_kernel_sizes": [3, 7, 11],
    "resblock_dilation_sizes": [[1, 3], [1, 3], [1, 3]],
    "num_mels": 80, "hop_size": 240, "sampling_rate": 24000,
}

FREGAN_CONFIG = {
    "resblock": "1", "seed": 1234,
    "upsample_rates": [5, 5, 2, 2, 2], "upsample_kernel_sizes": [10, 10, 4, 4, 4],
    "upsample_initial_channel": 512, "resblock_kernel_sizes": [3, 7, 11],
    "resblock_dilation_sizes": [[1, 3, 5, 7], [1, 3, 5, 7], [1, 3, 5, 7]],
    "num_mels": 80, "hop_size": 200, "sampling_rate": 16000,
}


def rescale_variance_preserving(sd: Dict[str, torch.Tensor], gain: float, seed: int = 7) -> Dict[str, torch.Tensor]:
    """A second, harder parity init: re-draw every conv weight with std = gain/sqrt(fan_in) and
    N(0,0.05) biases so activations stay O(1) through the stack like a trained model's."""
    import math

    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in sd.items():
        if k.endswith(".weight"):
            if k.startswith("ups.") or k.startswith("cond_up."):
                # ConvTranspose1d [Cin, Cout, K]: each output sees Cin*K/stride taps
                stride = max(1, v.shape[2] // 2)
                fan_in = v.shape[0] * v.shape[2] / stride
            else:
                fan_in = v.shape[1] * v.shape[2]
            out[k] = torch.randn(v.shape, generator=g) * (gain / math.sqrt(fan_in))
        else:
            out[k] = torch.randn(v.shape, generator=g) * 0.05
    return out


# ---- WaveRNN (fatchord_version.py:88-116; hparams models/vocoder/wavernn/hparams.py) ----------
WAVERNN_HP = dict(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 8), feat_dims=80,
                  compute_dims=128, res_out_dims=128, res_blocks=10, hop_length=256, sample_rate=16000,
                  mu_law=True, apply_preemphasis=True, preemphasis=0.97, mel_max_abs_value=4.0)


def wavernn_state_dict(seed: int = 0, randomize_bn: bool = True, mode: str = "RAW") -> Dict[str, torch.Tensor]:
    """``torch.manual_seed(seed); WaveRNN(..., mode=mode)`` state_dict, rebuilt from stock torch layers in the
    reference's construction order (UpsampleNetwork -> I -> rnn1 -> rnn2 -> fc1..3; fc3 has 2**bits outputs in mode
    'RAW', 30 in mode 'MOL', fatchord_version.py:95-100).  With
    ``randomize_bn`` the BatchNorm affine parameters and running statistics (which a fresh module
    leaves at identity) are overwritten from a side generator so that parity cases exercise them;
    oracle/make_golden.py applies the same overwrite to the live reference module."""
    hp = WAVERNN_HP
    torch.manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    cd, fd, ro = hp["compute_dims"], hp["feat_dims"], hp["res_out_dims"]
    k = hp["pad"] * 2 + 1
    sd["upsample.resnet.conv_in.weight"] = torch.nn.Conv1d(fd, cd, k, bias=False).weight.detach()
    bns = ["upsample.resnet.batch_norm"]
    for i in range(hp["res_blocks"]):
        sd[f"upsample.resnet.layers.{i}.conv1.weight"] = torch.nn.Conv1d(cd, cd, 1, bias=False).weight.detach()
        sd[f"upsample.resnet.layers.{i}.conv2.weight"] = torch.nn.Conv1d(cd, cd, 1, bias=False).weight.detach()
        bns += [f"upsample.resnet.layers.{i}.batch_norm1", f"upsample.resnet.layers.{i}.batch_norm2"]
    co = torch.nn.Conv1d(cd, ro, 1)
    sd["upsample.resnet.conv_out.weight"], sd["upsample.resnet.conv_out.bias"] = co.weight.detach(), co.bias.detach()
    for j, s in enumerate(hp["upsample_factors"]):
        c2 = torch.nn.Conv2d(1, 1, (1, 2 * s + 1), padding=(0, s), bias=False)  # consumes RNG, then filled
        sd[f"upsample.up_layers.{2 * j + 1}.weight"] = torch.full_like(c2.weight.detach(), 1.0 / (2 * s + 1))
    aux = ro // 4
    lin = torch.nn.Linear(fd + aux + 1, hp["rnn_dims"])
    sd["I.weight"], sd["I.bias"] = lin.weight.detach(), lin.bias.detach()
    for name, insz in (("rnn1", hp["rnn_dims"]), ("rnn2", hp["rnn_dims"] + aux)):
        g = torch.nn.GRU(insz, hp["rnn_dims"], batch_first=True)
        for p in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"):
            sd[f"{name}.{p}"] = getattr(g, p).detach()
    for name, insz, outsz in (("fc1", hp["rnn_dims"] + aux, hp["fc_dims"]), ("fc2", hp["fc_dims"] + aux, hp["fc_dims"]),
                              ("fc3", hp["fc_dims"], 2 ** hp["bits"] if mode == "RAW" else 30)):
        lin = torch.nn.Linear(insz, outsz)
        sd[f"{name}.weight"], sd[f"{name}.bias"] = lin.weight.detach(), lin.bias.detach()
    sd["step"] = torch.zeros(1).long()
    for b in bns:
        sd[b + ".weight"], sd[b + ".bias"] = torch.ones(cd), torch.zeros(cd)
        sd[b + ".running_mean"], sd[b + ".running_var"] = torch.zeros(cd), torch.ones(cd)
        sd[b + ".num_batches_tracked"] = torch.tensor(0)
    if randomize_bn:
        randomize_batchnorm_(sd, seed)
    return sd


def randomize_batchnorm_(sd: Dict[str, torch.Tensor], seed: int) -> None:
    g = torch.Generator().manual_seed(10_000 + seed)
    for k in sorted(sd):
        if k.endswith(".running_var"):
            sd[k] = torch.rand(sd[k].shape, generator=g) * 1.5 + 0.25
        elif k.endswith(".running_mean"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.3
        elif "batch_norm" in k and k.endswith(".weight"):
            sd[k] = torch.rand(sd[k].shape, generator=g) + 0.5
        elif "batch_norm" in k and k.endswith(".bias"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 0.2
    # learned FIR taps are Parameters too (SURVEY.md appendix A.3): perturb them off the box filter
    for k in sorted(sd):
        if k.startswith("upsample.up_layers."):
            sd[k] = sd[k] * (1.0 + 0.3 * torch.randn(sd[k].shape, generator=g))


def wavernn_noise(seed: int, B: int, steps: int) -> torch.Tensor:
    """The Exp(1) stream WaveRNN.generate consumes from the global torch generator under
    ``torch.manual_seed(seed)`` (SURVEY.md fact 5): two nn.GRUCell constructions
    (fatchord_version.py:160-161, 265-271) and then one exponential_([B,512]) per step (:223-226)."""
    torch.manual_seed(seed)
    torch.nn.GRUCell(512, 512)
    torch.nn.GRUCell(544, 512)
    out = torch.empty(steps, B, 512)
    for i in range(steps):
        out[i] = torch.empty(B, 512).exponential_(1)
    return out


def wavernn_mol_uniforms(seed: int, B: int, steps: int) -> torch.Tensor:
    """The uniform stream WaveRNN.generate consumes in mode 'MOL' under ``torch.manual_seed(seed)``: two nn.GRUCell
    constructions, then per step ``uniform_(1e-5, 1 - 1e-5)`` over [1, B, 10] (mixture pick) and over [1, B] (logistic
    draw), distribution.py:106, :117.  Returns [steps, 11 * B]."""
    torch.manual_seed(seed)
    torch.nn.GRUCell(512, 512)
    torch.nn.GRUCell(544, 512)
    out = torch.empty(steps, 11 * B)
    for i in range(steps):
        out[i, :10 * B] = torch.empty(1, B, 10).uniform_(1e-5, 1.0 - 1e-5).flatten()
        out[i, 10 * B:] = torch.empty(1, B).uniform_(1e-5, 1.0 - 1e-5).flatten()
    return out


# ---- Tacotron (models/synthesizer/models/tacotron.py:140-162; hparams models/synthesizer/hparams.py) ----
TACOTRON_HP = dict(embed_dims=512, num_chars=75, encoder_dims=256, decoder_dims=128, n_mels=80, fft_bins=80,
                   postnet_dims=512, encoder_K=5, lstm_dims=1024, postnet_K=5, num_highways=4, dropout=0.5,
                   stop_threshold=-3.4, speaker_embedding_size=256, gst_E=512, gst_token_num=10, gst_heads=8,
                   gst_ref_filters=(32, 32, 64, 64, 128, 128), gst_n_mels=256, max_r=20)


def _cbhg_modules(sd, prefix, K, in_channels, channels, proj_channels, num_highways):
    """CBHG.__init__ construction order (sublayer/cbhg.py:7-41)"""
    nn = torch.nn

    def bnconv(name, cin, cout, k):
        sd[f"{name}.conv.weight"] = nn.Conv1d(cin, cout, k, bias=False).weight.detach()
        bn = nn.BatchNorm1d(cout)
        for leaf in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked"):
            sd[f"{name}.bnorm.{leaf}"] = getattr(bn, leaf).detach().clone()

    for i, k in enumerate(range(1, K + 1)):
        bnconv(f"{prefix}.conv1d_bank.{i}", in_channels, channels, k)
    bnconv(f"{prefix}.conv_project1", K * channels, proj_channels[0], 3)
    bnconv(f"{prefix}.conv_project2", proj_channels[0], proj_channels[1], 3)
    if proj_channels[-1] != channels:
        sd[f"{prefix}.pre_highway.weight"] = nn.Linear(proj_channels[-1], channels, bias=False).weight.detach()
    for i in range(num_highways):
        w1, w2 = nn.Linear(channels, channels), nn.Linear(channels, channels)
        sd[f"{prefix}.highways.{i}.W1.weight"], sd[f"{prefix}.highways.{i}.W1.bias"] = w1.weight.detach(), torch.zeros(channels)
        sd[f"{prefix}.highways.{i}.W2.weight"], sd[f"{prefix}.highways.{i}.W2.bias"] = w2.weight.detach(), w2.bias.detach()
    g = nn.GRU(channels, channels // 2, batch_first=True, bidirectional=True)
    for n, p in g.named_parameters():
        sd[f"{prefix}.rnn.{n}"] = p.detach()


def tacotron_state_dict(seed: int = 0, r: int = 2, randomize_bn: bool = True) -> Dict[str, torch.Tensor]:
    """``torch.manual_seed(seed); Tacotron(**hparams)`` state_dict rebuilt from stock torch layers in the
    reference's construction order; ``decoder.r`` (a loaded buffer, tacotron.py:53) set to ``r``."""
    nn = torch.nn
    hp = TACOTRON_HP
    torch.manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def lin(name, i, o, bias=True):
        m = nn.Linear(i, o, bias=bias)
        sd[name + ".weight"] = m.weight.detach()
        if bias:
            sd[name + ".bias"] = m.bias.detach()

    # Encoder (tacotron.py:11-29)
    sd["encoder.embedding.weight"] = nn.Embedding(hp["num_chars"], hp["embed_dims"]).weight.detach()
    lin("encoder.pre_net.fc1", hp["embed_dims"], hp["encoder_dims"])
    lin("encoder.pre_net.fc2", hp["encoder_dims"], hp["encoder_dims"])
    _cbhg_modules(sd, "encoder.cbhg", hp["encoder_K"], hp["encoder_dims"], hp["encoder_dims"],
                  [hp["encoder_dims"], hp["encoder_dims"]], hp["num_highways"])
    project_dims = hp["encoder_dims"] + hp["speaker_embedding_size"] + hp["gst_E"]
    lin("encoder_proj", project_dims, hp["decoder_dims"], bias=False)
    # GlobalStyleToken (sublayer/global_style_token.py:9-96)
    filters = [1] + list(hp["gst_ref_filters"])
    convs = [nn.Conv2d(filters[i], filters[i + 1], (3, 3), (2, 2), (1, 1)) for i in range(len(filters) - 1)]
    for i, c in enumerate(convs):
        sd[f"gst.encoder.convs.{i}.weight"], sd[f"gst.encoder.convs.{i}.bias"] = c.weight.detach(), c.bias.detach()
    for i, f in enumerate(hp["gst_ref_filters"]):
        bn = nn.BatchNorm2d(f)
        for leaf in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked"):
            sd[f"gst.encoder.bns.{i}.{leaf}"] = getattr(bn, leaf).detach().clone()
    L = hp["gst_n_mels"]
    for _ in convs:
        L = (L - 3 + 2) // 2 + 1
    g = nn.GRU(hp["gst_ref_filters"][-1] * L, hp["gst_E"] // 2, batch_first=True)
    for n, p in g.named_parameters():
        sd[f"gst.encoder.gru.{n}"] = p.detach()
    d_q = hp["gst_E"] // 2 + hp["speaker_embedding_size"]
    d_k = hp["gst_E"] // hp["gst_heads"]
    lin("gst.stl.attention.W_query", d_q, hp["gst_E"], bias=False)
    lin("gst.stl.attention.W_key", d_k, hp["gst_E"], bias=False)
    lin("gst.stl.attention.W_value", d_k, hp["gst_E"], bias=False)
    sd["gst.stl.embed"] = torch.empty(hp["gst_token_num"], d_k).normal_(0, 0.5)
    # Decoder (tacotron.py:50-65)
    lin("decoder.prenet.fc1", hp["n_mels"], hp["decoder_dims"] * 2)
    lin("decoder.prenet.fc2", hp["decoder_dims"] * 2, hp["decoder_dims"] * 2)
    c = nn.Conv1d(1, 32, 31, padding=15)
    sd["decoder.attn_net.conv.weight"], sd["decoder.attn_net.conv.bias"] = c.weight.detach(), c.bias.detach()
    lin("decoder.attn_net.L", 32, hp["decoder_dims"], bias=False)
    lin("decoder.attn_net.W", hp["decoder_dims"], hp["decoder_dims"])
    lin("decoder.attn_net.v", hp["decoder_dims"], 1, bias=False)
    cell = nn.GRUCell(project_dims + hp["decoder_dims"] * 2, hp["decoder_dims"])
    for n, p in cell.named_parameters():
        sd[f"decoder.attn_rnn.{n}"] = p.detach()
    lin("decoder.rnn_input", project_dims + hp["decoder_dims"], hp["lstm_dims"])
    for name in ("res_rnn1", "res_rnn2"):
        cell = nn.LSTMCell(hp["lstm_dims"], hp["lstm_dims"])
        for n, p in cell.named_parameters():
            sd[f"decoder.{name}.{n}"] = p.detach()
    lin("decoder.mel_proj", hp["lstm_dims"], hp["n_mels"] * hp["max_r"], bias=False)
    lin("decoder.stop_proj", project_dims + hp["lstm_dims"], 1)
    sd["decoder.r"] = torch.tensor(r, dtype=torch.int)
    # postnet (tacotron.py:160-162)
    _cbhg_modules(sd, "postnet", hp["postnet_K"], hp["n_mels"], hp["postnet_dims"], [hp["postnet_dims"], hp["fft_bins"]],
                  hp["num_highways"])
    lin("post_proj", hp["postnet_dims"], hp["fft_bins"], bias=False)
    sd["step"] = torch.zeros(1, dtype=torch.long)
    sd["stop_threshold"] = torch.tensor(hp["stop_threshold"], dtype=torch.float32)
    if randomize_bn:
        g2 = torch.Generator().manual_seed(20_000 + seed)
        for k in sorted(sd):
            if ".bnorm." in k or ".bns." in k:
                if k.endswith(".running_var"):
                    sd[k] = torch.rand(sd[k].shape, generator=g2) * 1.5 + 0.25
                elif k.endswith(".running_mean"):
                    sd[k] = torch.randn(sd[k].shape, generator=g2) * 0.3
                elif k.endswith(".weight"):
                    sd[k] = torch.rand(sd[k].shape, generator=g2) + 0.5
                elif k.endswith(".bias"):
                    sd[k] = torch.randn(sd[k].shape, generator=g2) * 0.2
    return sd


def encoder_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """``torch.manual_seed(seed); SpeakerEncoder(cpu, cpu)`` state_dict rebuilt from stock torch layers in
    the reference's construction order (models/encoder/model.py:17-28): nn.LSTM(40, 256, 3), nn.Linear(256, 256);
    similarity_weight / similarity_bias are constants (10, -5) and consume no RNG."""
    nn = torch.nn
    torch.manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    lstm = nn.LSTM(input_size=40, hidden_size=256, num_layers=3, batch_first=True)
    for k, v in lstm.state_dict().items():
        sd["lstm." + k] = v.detach()
    lin = nn.Linear(256, 256)
    sd["linear.weight"], sd["linear.bias"] = lin.weight.detach(), lin.bias.detach()
    sd["similarity_weight"] = torch.tensor([10.0])
    sd["similarity_bias"] = torch.tensor([-5.0])
    return sd


# ---- DeepMind-style dual-softmax WaveRNN (models/vocoder/wavernn/models/deepmind_version.py:8-34) ----------------
def deepmind_state_dict(seed: int = 0, bias_scale: float = 0.1) -> Dict[str, torch.Tensor]:
    """``torch.manual_seed(seed); WaveRNN(hidden_size=896, quantisation=256)`` state_dict in the constructor's order
    (R, O1..O4, I_coarse, I_fine, then zero gate biases).  ``bias_scale`` > 0 additionally draws the three gate biases
    (zeros in a fresh module) from N(0, bias_scale) AFTER everything else, so that the fixtures exercise them."""
    torch.manual_seed(seed)
    nn = torch.nn
    H, S, Q = 896, 448, 256
    sd: Dict[str, torch.Tensor] = {}
    sd["R.weight"] = nn.Linear(H, 3 * H, bias=False).weight.detach()
    for name, (i, o) in (("O1", (S, S)), ("O2", (S, Q)), ("O3", (S, S)), ("O4", (S, Q))):
        m = nn.Linear(i, o)
        sd[name + ".weight"], sd[name + ".bias"] = m.weight.detach(), m.bias.detach()
    sd["I_coarse.weight"] = nn.Linear(2, 3 * S, bias=False).weight.detach()
    sd["I_fine.weight"] = nn.Linear(3, 3 * S, bias=False).weight.detach()
    for b in ("bias_u", "bias_r", "bias_e"):
        sd[b] = torch.zeros(H)
    if bias_scale > 0:
        for b in ("bias_u", "bias_r", "bias_e"):
            sd[b] = torch.randn(H) * bias_scale
    return sd


# ---- ppg2mel MelDecoderMOLv2 (models/ppg2mel/__init__.py:20-118, rnn_decoder_mol.py:24-107) ----------------------
PPG2MEL_CONFIG = dict(num_speakers=1, spk_embed_dim=256, bottle_neck_feature_dim=144, encoder_dim=256,
                      encoder_downsample_rates=[2, 2], attention_rnn_dim=512, decoder_rnn_dim=512, num_decoder_rnn_layer=1,
                      concat_context_to_last=True, prenet_dims=[256, 128], num_mixtures=5, frames_per_step=2,
                      mask_padding=True)


def ppg2mel_state_dict(seed: int = 0, randomize_bn: bool = True, bnf_dim: int = 144,
                       spk_dim: int = 256) -> Dict[str, torch.Tensor]:
    """``torch.manual_seed(seed); MelDecoderMOLv2(**PPG2MEL_CONFIG)`` state_dict rebuilt from stock torch layers in the
    constructor's order (``bnf_dim`` / ``spk_dim``: the config's bottle_neck_feature_dim / spk_embed_dim).  The reference's ``Linear`` / ``Conv1d`` wrappers (utils/basic_layers.py:27-56) build the
    torch layer (default init) and then redraw the weight with xavier_uniform_; MOLAttention.initialize_bias
    (utils/mol_attention.py:41-54) overwrites the sigma / Delta biases with constants (r = 2/4 < 1: Delta = -0.432).
    ``randomize_bn`` replaces the postnet BatchNorm statistics and affines (identity in a fresh module) by seeded draws."""
    nn = torch.nn
    gain = nn.init.calculate_gain
    torch.manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def put(name, m):
        for n, p in m.state_dict().items():
            sd[f"{name}.{n}"] = p.detach().clone()

    for branch, cin in (("bnf_prenet", bnf_dim), ("pitch_convs", 2)):
        put(f"{branch}.0", nn.Conv1d(cin, 256, 1, bias=False))
        put(f"{branch}.3", nn.Conv1d(256, 256, 4, 2, 1))
        put(f"{branch}.6", nn.Conv1d(256, 256, 4, 2, 1))
    put("reduce_proj", nn.Linear(256 + spk_dim, 256))

    def xlinear(name, i, o, bias=True, g="linear"):
        m = nn.Linear(i, o, bias=bias)
        nn.init.xavier_uniform_(m.weight, gain=gain(g))
        put(name + ".linear_layer", m)

    for pre in ("prenet", "prenet_pitch"):
        xlinear(f"decoder.{pre}.layers.0", 80, 256, bias=False)
        xlinear(f"decoder.{pre}.layers.1", 256, 128, bias=False)
    put("decoder.attention_rnn", nn.LSTMCell(384, 512))
    q0, q2 = nn.Linear(512, 256), nn.Linear(256, 15)
    with torch.no_grad():
        q2.bias[5:10] = 1.0
        q2.bias[10:15] = -0.432
    put("decoder.attention_layer.query_layer.0", q0)
    put("decoder.attention_layer.query_layer.2", q2)
    put("decoder.decoder_rnn_layers.0", nn.LSTMCell(768, 512))
    xlinear("decoder.linear_projection", 768, 160)
    xlinear("decoder.stop_layer", 768, 1, g="sigmoid")
    chans = [80, 512, 512, 512, 512, 80]
    for i in range(5):
        c = nn.Conv1d(chans[i], chans[i + 1], 5, 1, 2)
        nn.init.xavier_uniform_(c.weight, gain=gain("tanh" if i < 4 else "linear"))
        put(f"postnet.convolutions.{i}.0.conv", c)
        put(f"postnet.convolutions.{i}.1", nn.BatchNorm1d(chans[i + 1]))
    if randomize_bn:
        g2 = torch.Generator().manual_seed(30_000 + seed)
        for k in sorted(sd):
            if k.startswith("postnet.") and ".1." in k:
                if k.endswith(".running_var"):
                    sd[k] = torch.rand(sd[k].shape, generator=g2) * 1.5 + 0.25
                elif k.endswith(".running_mean"):
                    sd[k] = torch.randn(sd[k].shape, generator=g2) * 0.3
                elif k.endswith(".weight"):
                    sd[k] = torch.rand(sd[k].shape, generator=g2) + 0.5
                elif k.endswith(".bias"):
                    sd[k] = torch.randn(sd[k].shape, generator=g2) * 0.2
    return sd


# ---- PPG extractor (models/ppg_extractor/__init__.py:66-72: UtteranceMVN, DefaultFrontend, ConformerEncoder) ----------
# The released extractor's yaml is not in the reference tree: a stand-in in the reference's `args` layout.  D = 144 is
# ppg2mel's bottle_neck_feature_dim; 100 Hz frames without subsampling pair one to one with pyworld's 10 ms lf0_uv.
PPGX_CONFIG = dict(
    frontend_conf=dict(fs=16000, n_fft=400, win_length=400, hop_length=160, fmin=0, fmax=8000, n_mels=80),
    normalize_conf=dict(norm_means=True, norm_vars=True),
    encoder_conf=dict(attention_dim=144, attention_heads=4, linear_units=576, num_blocks=16, input_layer="conv2d",
                      no_subsample=True, macaron_style=True, pos_enc_layer_type="rel_pos",
                      selfattention_layer_type="rel_selfattn", activation_type="swish", use_cnn_module=True,
                      cnn_module_kernel=15))


def _ppgx_variant(base: dict, frontend=None, normalize=None, **enc) -> dict:
    return dict(frontend_conf=dict(base["frontend_conf"], **(frontend or {})),
                normalize_conf=dict(base["normalize_conf"], **(normalize or {})),
                encoder_conf=dict(base["encoder_conf"], **enc))


# test-only small config and variants reaching every supported option
PPGX_CONFIG_SMALL = _ppgx_variant(PPGX_CONFIG, attention_dim=32, attention_heads=2, linear_units=64, num_blocks=2,
                                  cnn_module_kernel=7)
PPGX_SMALL_VARIANTS = {
    "sub4": _ppgx_variant(PPGX_CONFIG_SMALL, no_subsample=False),
    "sub2": _ppgx_variant(PPGX_CONFIG_SMALL, no_subsample=False, subsample_by_2=True),
    "abs_pos": _ppgx_variant(PPGX_CONFIG_SMALL, pos_enc_layer_type="abs_pos", selfattention_layer_type="selfattn"),
    "plain": _ppgx_variant(PPGX_CONFIG_SMALL, macaron_style=False, use_cnn_module=False, activation_type="relu"),
    "no_vars": _ppgx_variant(PPGX_CONFIG_SMALL, normalize=dict(norm_vars=False)),
    "fft512": _ppgx_variant(PPGX_CONFIG_SMALL, frontend=dict(n_fft=512, win_length=400)),
    "vars_only": _ppgx_variant(PPGX_CONFIG_SMALL, normalize=dict(norm_means=False, norm_vars=True)),
    # frontend_conf without the STFT keys: DefaultFrontend's defaults n_fft 1024, win_length 800, hop_length 160
    "fe_defaults": dict(frontend_conf=dict(fs=16000, fmin=0, fmax=8000, n_mels=80),
                        normalize_conf=dict(PPGX_CONFIG_SMALL["normalize_conf"]),
                        encoder_conf=dict(PPGX_CONFIG_SMALL["encoder_conf"])),
}


def ppgx_frames(cfg: dict, n_samples: int) -> int:
    """PPG frames of an n-sample utterance: 1 + n // hop STFT frames (center=True; DefaultFrontend's default hop is
    160), halved by each stride-2 conv"""
    t = 1 + n_samples // cfg["frontend_conf"].get("hop_length", 160)
    enc = cfg["encoder_conf"]
    if not enc.get("no_subsample", False):
        t //= 2
        if not enc.get("subsample_by_2", False):
            t //= 2
    return t


def ppg_extractor_state_dict(cfg: dict, seed: int = 0, randomize_bn: bool = True) -> Dict[str, torch.Tensor]:
    """``torch.manual_seed(seed); build_model(argparse.Namespace(**cfg)).state_dict()`` rebuilt from stock torch layers in
    the constructor's order (encoder/conformer_encoder.py:80-200, subsampling.py, attention.py, convolution.py).  The
    melmat buffer is the current librosa meaning of ``norm=1`` (mockingbird_b200.synthesizer.audio_host.ppg_melmat).
    ``randomize_bn`` replaces the conv-module BatchNorm statistics and affines (identity in a fresh module) by seeded draws."""
    import numpy as np

    from mockingbird_b200.synthesizer.audio_host import ppg_melmat

    nn = torch.nn
    fe, enc = cfg["frontend_conf"], cfg["encoder_conf"]
    D, H, U = enc["attention_dim"], enc["attention_heads"], enc["linear_units"]
    n_mels = fe.get("n_mels", 80)
    fs = fe["fs"]  # DefaultFrontend has no default for it
    torch.manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def put(name, m):
        for n, p in m.state_dict().items():
            sd[f"{name}.{n}"] = p.detach().clone()

    mel = ppg_melmat(fs, fe.get("n_fft", 1024), n_mels, fe.get("fmin") or 0.0,
                     fe["fmax"] if fe.get("fmax") is not None else fs / 2, norm=fe.get("norm", 1))
    sd["frontend.logmel.melmat"] = torch.from_numpy(mel).float()
    sd["frontend.logmel.inv_melmat"] = torch.from_numpy(np.linalg.pinv(mel.T).T).float()
    if enc.get("no_subsample", False):
        convs, f_out = [(1, 5, 1, 2), (D, 5, 1, 2)], n_mels
    elif enc.get("subsample_by_2", False):
        convs, f_out = [(1, 5, 1, 2), (D, 4, 2, 1)], n_mels // 2
    else:
        convs, f_out = [(1, 4, 2, 1), (D, 4, 2, 1)], n_mels // 4
    for i, (cin, k, s, p) in zip((0, 2), convs):
        put(f"encoder.embed.conv.{i}", nn.Conv2d(cin, D, k, s, p))
    put("encoder.embed.out.0", nn.Linear(D * f_out, D))
    rel = enc.get("selfattention_layer_type", "selfattn") == "rel_selfattn"
    for b in range(enc["num_blocks"]):
        pre = f"encoder.encoders.{b}"
        att = {n: nn.Linear(D, D) for n in ("linear_q", "linear_k", "linear_v", "linear_out")}
        if rel:
            att["linear_pos"] = nn.Linear(D, D, bias=False)
            u, v = torch.empty(H, D // H), torch.empty(H, D // H)
            nn.init.xavier_uniform_(u)
            nn.init.xavier_uniform_(v)
            sd[f"{pre}.self_attn.pos_bias_u"], sd[f"{pre}.self_attn.pos_bias_v"] = u, v
        for n, m in att.items():
            put(f"{pre}.self_attn.{n}", m)
        ffs = ["feed_forward"] + (["feed_forward_macaron"] if enc.get("macaron_style", False) else [])
        for n in ffs:
            put(f"{pre}.{n}.w_1", nn.Linear(D, U))
            put(f"{pre}.{n}.w_2", nn.Linear(U, D))
        cnn = enc.get("use_cnn_module", False)
        if cnn:
            K = enc.get("cnn_module_kernel", 31)
            put(f"{pre}.conv_module.pointwise_conv1", nn.Conv1d(D, 2 * D, 1))
            put(f"{pre}.conv_module.depthwise_conv", nn.Conv1d(D, D, K, padding=(K - 1) // 2, groups=D))
            put(f"{pre}.conv_module.norm", nn.BatchNorm1d(D))
            put(f"{pre}.conv_module.pointwise_conv2", nn.Conv1d(D, D, 1))
        norms = ["norm_ff", "norm_mha"] + (["norm_ff_macaron"] if len(ffs) == 2 else []) + \
            (["norm_conv", "norm_final"] if cnn else [])
        for n in norms:
            put(f"{pre}.{n}", nn.LayerNorm(D, eps=1e-12))
    put("encoder.after_norm", nn.LayerNorm(D, eps=1e-12))
    if randomize_bn:
        g2 = torch.Generator().manual_seed(40_000 + seed)
        for k in sorted(sd):
            if ".conv_module.norm." in k:
                if k.endswith(".running_var"):
                    sd[k] = torch.rand(sd[k].shape, generator=g2) * 1.5 + 0.25
                elif k.endswith(".running_mean"):
                    sd[k] = torch.randn(sd[k].shape, generator=g2) * 0.3
                elif k.endswith(".weight"):
                    sd[k] = torch.rand(sd[k].shape, generator=g2) + 0.5
                elif k.endswith(".bias"):
                    sd[k] = torch.randn(sd[k].shape, generator=g2) * 0.2
    return sd


# ---- VITS (models/synthesizer/models/vits.py:389-456), inference modules only ------------------------------------------
# Two stand-in configurations: the reference tree ships no VITS config or checkpoint.  VITS_CONFIG is the usual VITS shape
# (multi-speaker, gin_channels = 256); VITS_TOY a small one for fast tests.
VITS_CONFIG = dict(n_vocab=80, spec_channels=513, segment_size=32, inter_channels=192, hidden_channels=192, filter_channels=768,
                   n_heads=2, n_layers=6, kernel_size=3, p_dropout=0.1, resblock="1", resblock_kernel_sizes=[3, 7, 11],
                   resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], upsample_rates=[8, 8, 2, 2],
                   upsample_initial_channel=512, upsample_kernel_sizes=[16, 16, 4, 4], n_speakers=4, gin_channels=256, use_sdp=True)
VITS_TOY = dict(n_vocab=20, spec_channels=33, segment_size=8, inter_channels=16, hidden_channels=16, filter_channels=32,
                n_heads=2, n_layers=2, kernel_size=3, p_dropout=0.1, resblock="2", resblock_kernel_sizes=[3, 5],
                resblock_dilation_sizes=[[1, 3], [1, 3]], upsample_rates=[4, 2], upsample_initial_channel=32,
                upsample_kernel_sizes=[8, 4], n_speakers=3, gin_channels=8, use_sdp=True)

# single speaker (no emb_g, no cond layers) with upsampling stages whose ConvTranspose1d padding (k-u)//2 differs from
# HiFi-GAN's u//2 + u%2
VITS_TOY_1SPK = dict(VITS_TOY, n_speakers=0, gin_channels=0, resblock="1", resblock_kernel_sizes=[3],
                     resblock_dilation_sizes=[[1, 3, 5]], upsample_rates=[4, 2], upsample_kernel_sizes=[12, 6])


def vits_state_dict(cfg: dict, seed: int = 0, gain: float = 1.0) -> Dict[str, torch.Tensor]:
    """Seeded random weights for ``Vits(**cfg)``'s inference modules (enc_p, emb_g, dp, flow, dec), with the reference's
    parameter names and shapes and folded ("weight") weight-norm tensors.  Every conv / linear weight is drawn with std
    gain / sqrt(fan_in) and every bias from N(0, 0.05): the variance-preserving rescale the GAN goldens use, so that neither
    the text encoder nor the decoder saturates.  ResidualCouplingLayer.post and ConvFlow.proj, zero at the reference's init,
    are drawn with std 0.1 / sqrt(fan_in) so that every flow does work.  LayerNorm gains are 1 + N(0, 0.05), the SDP's
    ElementwiseAffine N(0, 0.1)."""
    import math

    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    def conv(name, co, ci, k, bias=True, scale=1.0, fan=None):
        sd[name + ".weight"] = rn(co, ci, k, std=scale * gain / math.sqrt(fan or ci * k))
        if bias:
            sd[name + ".bias"] = rn(co, std=0.05)

    def ln(name, c):
        sd[name + ".gamma"] = 1 + rn(c, std=0.05)
        sd[name + ".beta"] = rn(c, std=0.05)

    I, H, F, K = cfg["inter_channels"], cfg["hidden_channels"], cfg["filter_channels"], cfg["kernel_size"]
    G, nh = cfg["gin_channels"], cfg["n_heads"]
    sd["enc_p.emb.weight"] = rn(cfg["n_vocab"], H, std=H ** -0.5)
    sd["enc_p.emo_proj.weight"] = rn(H, 1024, std=gain / math.sqrt(1024) * 0.5)
    sd["enc_p.emo_proj.bias"] = rn(H, std=0.05)
    for i in range(cfg["n_layers"]):
        a = f"enc_p.encoder.attn_layers.{i}"
        for c in ("conv_q", "conv_k", "conv_v", "conv_o"):
            conv(f"{a}.{c}", H, H, 1)
        sd[a + ".emb_rel_k"] = rn(1, 9, H // nh, std=(H // nh) ** -0.5)
        sd[a + ".emb_rel_v"] = rn(1, 9, H // nh, std=(H // nh) ** -0.5)
        ln(f"enc_p.encoder.norm_layers_1.{i}", H)
        conv(f"enc_p.encoder.ffn_layers.{i}.conv_1", F, H, K)
        conv(f"enc_p.encoder.ffn_layers.{i}.conv_2", H, F, K)
        ln(f"enc_p.encoder.norm_layers_2.{i}", H)
    conv("enc_p.proj", 2 * I, H, 1, scale=0.5)
    if cfg["n_speakers"] > 1:
        sd["emb_g.weight"] = rn(cfg["n_speakers"], G)

    def dds(name, c):
        for l in range(3):
            conv(f"{name}.convs_sep.{l}", c, 1, 3)
            conv(f"{name}.convs_1x1.{l}", c, c, 1)
            ln(f"{name}.norms_1.{l}", c)
            ln(f"{name}.norms_2.{l}", c)

    if cfg["use_sdp"]:
        conv("dp.pre", H, H, 1)
        conv("dp.proj", H, H, 1)
        dds("dp.convs", H)
        if G:
            conv("dp.cond", H, G, 1)
        sd["dp.flows.0.m"] = rn(2, 1, std=0.1)
        sd["dp.flows.0.logs"] = rn(2, 1, std=0.1)
        for f in (1, 3, 5, 7):
            conv(f"dp.flows.{f}.pre", H, 1, 1)
            dds(f"dp.flows.{f}.convs", H)
            conv(f"dp.flows.{f}.proj", 29, H, 1, scale=0.1)
    else:
        conv("dp.conv_1", 256, H, 3)
        ln("dp.norm_1", 256)
        conv("dp.conv_2", 256, 256, 3)
        ln("dp.norm_2", 256)
        conv("dp.proj", 1, 256, 1, scale=0.3)
        sd["dp.proj.bias"] += 1.0  # logw around 1: durations of 2-4 frames, not all ceil'ed to 1
        if G:
            conv("dp.cond", H, G, 1)
    for f in (0, 2, 4, 6):
        n = f"flow.flows.{f}"
        conv(n + ".pre", H, I // 2, 1)
        for l in range(4):
            conv(f"{n}.enc.in_layers.{l}", 2 * H, H, 5)
            conv(f"{n}.enc.res_skip_layers.{l}", 2 * H if l < 3 else H, H, 1)
        if G:
            conv(n + ".enc.cond_layer", 2 * H * 4, G, 1)
        conv(n + ".post", I // 2, H, 1, scale=0.1)
    C0 = cfg["upsample_initial_channel"]
    conv("dec.conv_pre", C0, I, 7)
    if G:
        conv("dec.cond", C0, G, 1)
    ch = C0
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        sd[f"dec.ups.{i}.weight"] = rn(ch, ch // 2, k, std=gain / math.sqrt(ch * k / u))
        sd[f"dec.ups.{i}.bias"] = rn(ch // 2, std=0.05)
        ch //= 2
        for j, (rk, ds) in enumerate(zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])):
            base = f"dec.resblocks.{i * len(cfg['resblock_kernel_sizes']) + j}"
            groups = ("convs1", "convs2") if str(cfg["resblock"]) == "1" else ("convs",)
            for grp in groups:
                for m in range(len(ds)):
                    conv(f"{base}.{grp}.{m}", ch, ch, rk, scale=0.5)
    conv("dec.conv_post", 1, ch, 7, bias=False)
    return sd


# ---- wav2vec2 emotion model (models/synthesizer/models/wav2emo.py EmotionExtractorModel) -----------------------------------
# The released checkpoint (audeering/wav2vec2-large-robust-12-ft-emotion-msp-dim) and its config.json are not in the
# reference tree.  WAV2EMO_CONFIG is a stand-in with that model's published shape, taken from its public model card and
# config: wav2vec2-large-robust pruned to 12 layers, hidden 1024, 16 heads, 4096 units, 128-tap positional conv in 16 groups,
# conv_bias, layer_norm_eps 1e-5, and 3 regression labels (arousal, dominance, valence).
WAV2EMO_CONFIG = dict(
    hidden_size=1024, num_hidden_layers=12, num_attention_heads=16, intermediate_size=4096,
    conv_dim=[512] * 7, conv_kernel=[10, 3, 3, 3, 3, 2, 2], conv_stride=[5, 2, 2, 2, 2, 2, 2], conv_bias=True,
    num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=16, layer_norm_eps=1e-5,
    feat_extract_norm="layer", do_stable_layer_norm=True, feat_extract_activation="gelu", hidden_act="gelu",
    add_adapter=False, num_labels=3, final_dropout=0.1, vocab_size=32,
)
WAV2EMO_CONFIG_SMALL = dict(WAV2EMO_CONFIG, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
                            conv_dim=[128] * 5, conv_kernel=[10, 3, 3, 2, 2], conv_stride=[5, 2, 2, 2, 2],
                            num_conv_pos_embeddings=16, num_conv_pos_embedding_groups=2)
WAV2EMO_SMALL_VARIANTS = {
    "nobias": dict(conv_bias=False),
    "oddpos": dict(num_conv_pos_embeddings=15),          # odd kernel: SamePad removes nothing
    "groups1": dict(num_conv_pos_embedding_groups=1),    # one 128-channel group
    "short": dict(conv_dim=[128] * 3, conv_kernel=[10, 3, 3], conv_stride=[5, 2, 2]),
    "onelabel": dict(num_labels=1, layer_norm_eps=1e-6),
}


def wav2emo_variant(name: str) -> dict:
    return dict(WAV2EMO_CONFIG_SMALL, **WAV2EMO_SMALL_VARIANTS[name])


def wav2emo_state_dict(cfg: dict, seed: int = 0) -> Dict[str, torch.Tensor]:
    """EmotionExtractorModel weights in transformers-5 key names (the positional conv's weight norm as
    parametrizations.weight.original0 / original1).  Variance-preserving linear and conv weights, LayerNorm affines away from
    (1, 0), small biases, and a classifier whose tanh input stays well inside (-1, 1), so every stage does work."""
    g = torch.Generator().manual_seed(seed)

    def normal(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    sd: Dict[str, torch.Tensor] = {}
    D, U = cfg["hidden_size"], cfg["intermediate_size"]

    def ln(name, n):
        sd[name + ".weight"] = 1.0 + normal(n, std=0.1)
        sd[name + ".bias"] = normal(n, std=0.1)

    def linear(name, n_out, n_in, gain=1.0):
        sd[name + ".weight"] = normal(n_out, n_in, std=gain / math.sqrt(n_in))
        sd[name + ".bias"] = normal(n_out, std=0.05)

    c_in = 1
    for i, (c, k) in enumerate(zip(cfg["conv_dim"], cfg["conv_kernel"])):
        b = f"wav2vec2.feature_extractor.conv_layers.{i}."
        sd[b + "conv.weight"] = normal(c, c_in, k, std=1.0 / math.sqrt(c_in * k))
        if cfg["conv_bias"]:
            sd[b + "conv.bias"] = normal(c, std=0.05)
        ln(b + "layer_norm", c)
        c_in = c
    ln("wav2vec2.feature_projection.layer_norm", c_in)
    linear("wav2vec2.feature_projection.projection", D, c_in)
    sd["wav2vec2.masked_spec_embed"] = torch.rand(D, generator=g)
    k, G = cfg["num_conv_pos_embeddings"], cfg["num_conv_pos_embedding_groups"]
    p = "wav2vec2.encoder.pos_conv_embed.conv."
    sd[p + "bias"] = normal(D, std=0.05)
    sd[p + "parametrizations.weight.original0"] = 0.5 + torch.rand(1, 1, k, generator=g) * math.sqrt(D / k)
    sd[p + "parametrizations.weight.original1"] = normal(D, D // G, k)
    ln("wav2vec2.encoder.layer_norm", D)
    for i in range(cfg["num_hidden_layers"]):
        b = f"wav2vec2.encoder.layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            linear(b + "attention." + n, D, D)
        ln(b + "layer_norm", D)
        linear(b + "feed_forward.intermediate_dense", U, D)
        linear(b + "feed_forward.output_dense", D, U)
        ln(b + "final_layer_norm", D)
    linear("classifier.dense", D, D, gain=2.0)
    linear("classifier.out_proj", cfg["num_labels"], D)
    # biases of magnitude 0.5..1 keep each logit away from zero, so its error is measured against a value the head produces
    # rather than against the cancellation of out_proj's terms
    n = cfg["num_labels"]
    sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
    sd["classifier.out_proj.bias"] = sign * (0.5 + 0.5 * torch.rand(n, generator=g))
    return sd
