"""CPU tests of the 24 kHz HiFi-GAN (nearest upsample + Conv1d per stage, hifigan/models.py:107-118).

Pins the seeded weights and the oracle against the live reference where it can be read (and the oracle against the committed
fixture everywhere), the nearest-index property the folded lowering relies on, the fold itself, the host-only plan of the
library (taps, tensor-core coverage, work) and the configs it rejects.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gan_oracle as go
import hifigan24k_oracle as o24
import ref_harness as rh
import ref_init as ri

needs_ref = pytest.mark.skipif(not rh.reference_available(), reason="reference tree not present")

CONFIGS = {"24k": ri.HIFIGAN_CONFIG_24K, "24k_u8": ri.HIFIGAN_CONFIG_24K_U8}
K_PAD_ROWS = 40  # gan_kernels.h kPadRows


def _reference(cfg, seed=0):
    from make_golden_hifigan24k import build_reference_24k

    return build_reference_24k(cfg, seed)


@needs_ref
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_ref_init_matches_reference_constructor(name):
    cfg = CONFIGS[name]
    ref = {k: v.detach() for k, v in _reference(cfg).state_dict().items()}
    sd = ri.hifigan_state_dict(cfg, 0)
    assert sorted(sd) == sorted(ref)
    assert any(k.startswith("ups.0.1.") for k in sd)
    for k in ref:
        assert torch.equal(sd[k], ref[k]), k


@needs_ref
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_oracle_matches_reference_forward(name):
    cfg = CONFIGS[name]
    g = _reference(cfg)
    sd = ri.hifigan_state_dict(cfg, 0)
    mel = torch.rand(2, 80, 9, generator=torch.Generator().manual_seed(5)) * 8 - 4
    with torch.no_grad():
        ref = g(mel)
        got = o24.hifigan24k_forward(sd, cfg, mel)
    assert ref.shape == (2, 1, 9 * 240)
    assert torch.equal(got, ref)


def test_oracle_reproduces_fixture(golden_dir):
    z = np.load(golden_dir / "hifigan24k_seed0.npz")
    cfg = ri.HIFIGAN_CONFIG_24K
    sd = ri.hifigan_state_dict(cfg, 0)
    mel_full = torch.rand(32, 80, 256, generator=torch.Generator().manual_seed(2)) * 8 - 4
    with torch.no_grad():
        small = o24.hifigan24k_forward(sd, cfg, torch.from_numpy(z["mel_small"]))
        full = torch.cat([o24.hifigan24k_forward(sd, cfg, mel_full[int(i):int(i) + 1]) for i in z["full_pick"]])
    assert small.shape == (2, 1, 24 * 240) and full.shape == (2, 1, 256 * 240)
    # same torch build: bit-identical; another CPU capability / thread count: last-ulp noise only
    for got, ref in ((small, z["wav_small"]), (full, z["wav_full"])):
        e = go.rel_errors(got, torch.from_numpy(ref))
        assert e["max_rel"] < 1e-5 and e["rms_rel"] < 1e-5, e


@pytest.mark.parametrize("u", range(1, 9))
def test_nearest_index_is_floor_division(u):
    """F.interpolate(size=L*u, mode='nearest', recompute_scale_factor=False) reads source row dst // u for every output row: torch
    takes floor(dst * fl(1/u)) and fl(1/u) >= 1/u for u <= 8 (a power of two is exact; 3, 5, 6, 7 round up), while
    dst * fl(1/u) stays below the next integer for dst < 2^20.  The folded lowering depends on it."""
    for L in (1, 2, 7, 255, 4096, (1 << 20) // u):
        x = torch.arange(L, dtype=torch.float64).view(1, 1, L)
        idx = o24.interpolate_nearest(x, u).view(-1).long()
        assert torch.equal(idx, torch.arange(L * u) // u), (u, L)


@pytest.mark.parametrize("u,k", [(5, 11), (4, 9), (3, 7), (2, 5), (8, 17), (8, 3), (2, 1), (1, 7), (7, 21), (3, 13)])
def test_fold_equals_interpolate_and_conv(u, k):
    g = torch.Generator().manual_seed(u * 100 + k)
    x = torch.randn(2, 6, 13, generator=g, dtype=torch.float64)
    w = torch.randn(5, 6, k, generator=g, dtype=torch.float64)
    b = torch.randn(5, generator=g, dtype=torch.float64)
    ref = F.conv1d(o24.interpolate_nearest(x, u), w, b, padding=(k - 1) // 2)
    assert ref.shape[-1] == 13 * u
    assert torch.allclose(o24.folded_forward(x, w, b, u), ref, rtol=1e-12, atol=1e-12)
    for taps in o24.fold_taps(u, k):
        ds = [d for d, _, _ in taps]
        assert ds == list(range(ds[0], ds[-1] + 1))


def test_fold_weight_norm_of_interpolation_convs():
    """ups.{i}.1 is a weight-normed Conv1d: weight_g has one entry per output channel (dim 0)"""
    from mockingbird_b200.vocoder._gan import fold_weight_norm

    torch.manual_seed(0)
    m = torch.nn.utils.weight_norm(torch.nn.Conv1d(6, 4, 5))
    with torch.no_grad():
        m.weight_g.mul_(torch.rand_like(m.weight_g) + 0.5)
    sd = {f"ups.0.1.{k}": v.detach() for k, v in m.state_dict().items()}
    assert sd["ups.0.1.weight_g"].shape == (4, 1, 1)
    torch.nn.utils.remove_weight_norm(m)
    out = fold_weight_norm(sd)
    assert sorted(out) == ["ups.0.1.bias", "ups.0.1.weight"]
    assert torch.allclose(out["ups.0.1.weight"], m.weight.detach(), rtol=1e-6, atol=1e-7)


# ---- the library's plan (host-only: mb_gan_create, mb_gan_tc_plan_info and mb_gan_layer_work need no GPU) ----------------

def _gen(cfg, precision):
    from mockingbird_b200.vocoder.hifigan.models import Generator

    return Generator(cfg, precision=precision)


def _layer(g, i):
    s = g.layer_info(i).split()
    return s[0], s[1], {k: int(v) for k, v in (t.split("=") for t in s[2:])}


@pytest.mark.parametrize("precision", ["f16tc", "f16x3", "fp32"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_plan_of_interpolation_layers(name, precision):
    from mockingbird_b200 import _lib

    cfg = CONFIGS[name]
    g = _gen(cfg, precision)
    assert g.kind == _lib.MB_GAN_HIFIGAN_INTERP and g.hop == 240
    ups = [(i, _layer(g, i)) for i in range(g.num_layers()) if _layer(g, i)[1].startswith("ups.")]
    assert [n for _, (_, n, _) in ups] == [f"ups.{i}.1" for i in range(len(cfg["upsample_rates"]))]
    C0 = cfg["upsample_initial_channel"]
    rate = 1
    for s, (i, (_, n, d)) in enumerate(ups):
        u, k = cfg["upsample_rates"][s], cfg["upsample_kernel_sizes"][s]
        assert d["stride"] == u and d["k"] == k and d["rate_in"] == rate, (n, d)
        rate *= u
        # folded work: 3 taps per output row of the checkpoint's channels (k * u / 3 less than interpolate + conv)
        macs, _ = g.layer_work(i, 1, 1)
        assert macs == rate * 3 * (C0 >> s) * (C0 >> (s + 1)), (n, macs)
        if precision == "fp32":
            continue
        p = g.tc_plan_info(i)
        assert p["use_tc"] == 1 and p["x3"] == 1, (n, p)  # the 3-term split in f16tc too, like the transposed ups
        assert (p["omin"], p["omax"]) == (-1, 1), (n, p)
        assert p["kernel"] == (d["cout"], p["mt"], 64, 0), (n, p)
    assert rate == 240


def test_plan_pads_the_16_channel_stage():
    g = _gen(ri.HIFIGAN_CONFIG_24K, "f16tc")
    for i in range(g.num_layers()):
        kind, n, d = _layer(g, i)
        if n == "ups.4.1":
            assert d["cin"] == 32 and d["cout"] == 32  # the checkpoint's 16 output channels carried as 32
        if n == "conv_post":
            assert d["cin"] == 32


def test_plan_kernels_are_compiled():
    from test_gan_tc_plan import compiled_instances

    inst = compiled_instances()
    for cfg in CONFIGS.values():
        for precision in ("f16tc", "f16x3"):
            g = _gen(cfg, precision)
            for i in range(g.num_layers()):
                if g.layer_info(i).startswith("conv"):
                    p = g.tc_plan_info(i)
                    if p["kernel"] != (0, 0, 0, 0):
                        assert p["kernel"] in inst, p
                        assert p["omin"] >= -K_PAD_ROWS and p["omax"] <= K_PAD_ROWS, p


@pytest.mark.parametrize("precision", ["f16tc", "fp32"])
def test_fregan_res_output_keeps_one_tap(precision):
    from mockingbird_b200.vocoder.fregan.models import FreGAN

    cfg = ri.FREGAN_CONFIG
    g = FreGAN(cfg, precision=precision)
    seen = 0
    for i in range(g.num_layers()):
        kind, n, d = _layer(g, i)
        if not n.startswith("res_output."):
            continue
        seen += 1
        macs, _ = g.layer_work(i, 1, 1)
        cin_w = cfg["upsample_initial_channel"] >> (int(n.split(".")[1]) + len(cfg["upsample_rates"]) - 4 + 1)
        assert d["k"] == 1 and macs == d["rate_in"] * d["stride"] * cin_w * (cin_w // 2), (n, d, macs)
        if precision != "fp32":
            p = g.tc_plan_info(i)
            assert (p["omin"], p["omax"]) == (0, 0) or p["kernel"] == (0, 0, 0, 0), (n, p)
    assert seen == 3


@pytest.mark.parametrize("change,match", [
    ({"upsample_kernel_sizes": [10, 9, 7, 5, 5]}, r"even k.*u\*L-1 samples"),
    ({"upsample_rates": [9, 4, 3, 2, 2]}, r"upsample rate 9"),
    ({"upsample_rates": [2, 4, 3, 2, 2], "upsample_kernel_sizes": [23, 9, 7, 5, 5]}, r"folds to 12 taps per phase"),
    ({"upsample_rates": [1, 4, 3, 2, 2], "upsample_kernel_sizes": [13, 9, 7, 5, 5]}, r"folds to 13 taps per phase"),
])
def test_rejected_configs(change, match):
    from mockingbird_b200 import _lib

    with pytest.raises(_lib.MbError, match=match):
        _gen(dict(ri.HIFIGAN_CONFIG_24K, **change), "f16tc")


def test_16k_generator_keeps_transposed_layers():
    from mockingbird_b200 import _lib

    g = _gen(ri.HIFIGAN_CONFIG_16K, "f16tc")
    assert g.kind == _lib.MB_GAN_HIFIGAN
    assert [_layer(g, i)[1] for i in range(g.num_layers()) if _layer(g, i)[1].startswith("ups.")] == ["ups.0", "ups.1", "ups.2", "ups.3"]
