"""CPU tests of the tensor-core execution plan (mb_gan_tc_plan_info is host-only, like mb_gan_create).

Pins which resblock pairs run as ONE fused launch (tc_conv_kernel<..., PAIR = true>), at which row tiles per work item (MT),
whether c1's weights stay resident in shared memory or stream through a ring, and that no op reads further than the planes'
kPadRows zero rows.  The table is the one in DESIGN.md 3.3.
"""
import re
from pathlib import Path

import pytest

import ref_init as ri

ROOT = Path(__file__).resolve().parent.parent
K_PAD_ROWS = 40  # gan_kernels.h kPadRows

# (C, k, dilation) -> (MT, rows per item, c1's weights resident, c1's weight stages)
FUSED = {
    (64, 3, 1): (2, 254, 1, 3), (64, 3, 3): (2, 254, 1, 3), (64, 3, 5): (2, 254, 1, 3), (64, 3, 7): (2, 254, 1, 3),
    (64, 7, 1): (2, 250, 0, 6), (64, 7, 3): (2, 250, 0, 5), (64, 7, 5): (2, 250, 0, 5), (64, 7, 7): (2, 250, 0, 4),
    (64, 11, 1): (1, 118, 0, 7), (64, 11, 3): (1, 118, 0, 7), (64, 11, 5): (1, 118, 0, 6), (64, 11, 7): (1, 118, 0, 5),
    (32, 3, 1): (8, 1022, 0, 2), (32, 3, 3): (8, 1022, 0, 2), (32, 3, 5): (4, 510, 1, 3), (32, 3, 7): (4, 510, 1, 3),
    (32, 7, 1): (4, 506, 1, 7), (32, 7, 3): (4, 506, 1, 7), (32, 7, 5): (4, 506, 1, 7), (32, 7, 7): (4, 506, 1, 7),
    (32, 11, 1): (4, 502, 1, 11), (32, 11, 3): (4, 502, 1, 11), (32, 11, 5): (4, 502, 1, 11), (32, 11, 7): (4, 502, 1, 11),
}
PAIR_KERNEL = {(64, 2): (64, 2, 64, 1), (64, 1): (64, 1, 64, 1), (32, 8): (32, 8, 32, 1), (32, 4): (32, 4, 32, 1)}

CONFIGS = {"hifigan": ri.HIFIGAN_CONFIG_16K, "fregan": ri.FREGAN_CONFIG}


def _gen(kind, precision):
    from mockingbird_b200.vocoder.fregan.models import FreGAN
    from mockingbird_b200.vocoder.hifigan.models import Generator

    return (Generator if kind == "hifigan" else FreGAN)(CONFIGS[kind], precision=precision)


def _layer(g, i):
    info = g.layer_info(i)
    d = {k: int(v) for k, v in (t.split("=") for t in info.split()[2:])}
    return info.split()[0], info.split()[1], d


def plan_rows(g):
    """[(op index, name, layer dict, plan dict)] of every conv"""
    out = []
    for i in range(g.num_layers()):
        kind, name, d = _layer(g, i)
        if kind == "conv":
            out.append((i, name, d, g.tc_plan_info(i)))
    return out


def compiled_instances():
    """the tc_conv_kernel instances gan_tc.cu compiles (its kTcInstances table)"""
    src = (ROOT / "mockingbird_b200" / "csrc" / "gan_tc.cu").read_text()
    found = re.findall(r"\{(\d+), (\d+), (\d+), (true|false), tc_conv_kernel<", src)
    return {(int(n), int(mt), int(cw), int(p == "true")) for n, mt, cw, p in found}


@pytest.mark.parametrize("kind", ["hifigan", "fregan"])
def test_f16tc_fused_pairs(kind):
    g = _gen(kind, "f16tc")
    rows = plan_rows(g)
    seen = set()
    for j, (i, name, d, p) in enumerate(rows):
        is_c1 = ".convs1." in name
        if is_c1 and d["cout"] in (32, 64):
            # every C = 32 / 64 resblock pair fuses, as the table says
            key = (d["cout"], d["k"], d["dil"])
            assert p["fuse_next"] == 1, (name, p)
            mt, rows_item, resident, wstages = FUSED[key]
            assert (p["pair_mt"], p["pair_rows_item"], p["pair_resident"], p["pair_wstages"]) == (mt, rows_item, resident, wstages), (name, p)
            assert p["pair_rows_item"] == 128 * p["pair_mt"] - 2 * ((d["k"] - 1) // 2)
            assert p["kernel"] == PAIR_KERNEL[(d["cout"], mt)], (name, p)
            assert p["pair_omin"] == -(d["k"] - 1) // 2 * d["dil"] - (d["k"] - 1) // 2
            nxt = rows[j + 1]
            assert ".convs2." in nxt[1] and nxt[3]["fused_prev"] == 1 and nxt[3]["kernel"] == (0, 0, 0, 0)
            seen.add(key)
        elif ".convs1." in name:
            assert p["fuse_next"] == 0 and d["cout"] >= 128, (name, p)
        if not p["fused_prev"] and ".convs2." in name:
            assert d["cout"] >= 128, (name, p)
    dils = {1, 3, 5} if kind == "hifigan" else {1, 3, 5, 7}
    assert seen == {k for k in FUSED if k[2] in dils}


@pytest.mark.parametrize("kind", ["hifigan", "fregan"])
def test_f16x3_runs_unfused(kind):
    """3-term-split layers run unfused; every tensor-core conv is an x3 layer (conv_pre: the fp32-input split)"""
    g = _gen(kind, "f16x3")
    for i, name, d, p in plan_rows(g):
        assert p["fuse_next"] == 0 and p["fused_prev"] == 0, (name, p)
        if p["use_tc"]:
            assert p["x3"] == 1 and p["kernel"][3] == 0, (name, p)
            assert p["kernel"] == (d["cout"], p["mt"], 64, 0)
        if ".convs" in name:
            assert p["use_tc"] == 1, (name, p)


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("kind", ["hifigan", "fregan"])
def test_taps_stay_inside_the_zero_padding(kind, precision):
    g = _gen(kind, precision)
    deepest = 0
    for i, name, d, p in plan_rows(g):
        if p["kernel"] == (0, 0, 0, 0):
            continue
        assert p["omin"] >= -K_PAD_ROWS and p["omax"] <= K_PAD_ROWS, (name, p)
        if p["fuse_next"]:
            assert p["pair_omin"] >= -K_PAD_ROWS, (name, p)
            deepest = min(deepest, p["pair_omin"])
    if kind == "fregan" and precision == "f16tc":
        assert deepest == -K_PAD_ROWS  # the k = 11, d = 7 pair: c1 at offsets -35 ... shifted by c2's halo of 5
    elif precision == "f16tc":
        assert deepest == -30


@pytest.mark.parametrize("precision", ["f16tc", "f16x3"])
@pytest.mark.parametrize("kind", ["hifigan", "fregan"])
def test_plan_kernels_are_compiled(kind, precision):
    inst = compiled_instances()
    assert len(inst) == 11
    g = _gen(kind, precision)
    for i, name, d, p in plan_rows(g):
        if p["kernel"] != (0, 0, 0, 0):
            assert p["kernel"] in inst, (name, p)


def test_design_table_matches():
    """DESIGN.md 3.3's fusion table states the pinned plan"""
    text = (ROOT / "DESIGN.md").read_text()
    for (c, k), (mt, rows_item) in {(64, 3): (2, 254), (64, 7): (2, 250), (64, 11): (1, 118), (32, 3): (8, 1022),
                                    (32, 7): (4, 506), (32, 11): (4, 502)}.items():
        assert FUSED[(c, k, 1)][:2] == (mt, rows_item)
        assert re.search(rf"\| {c} \| [^|]*\b{k}\b[^|]* \|[^|]*\| {mt} \| [^|]*\b{rows_item}\b", text), (c, k)
    assert "C = 64, k = 11) runs as two" not in text


def test_pair_checker_is_sharp():
    """the fused-pair checker (oracle/tc_pair_oracle.py) accepts an fp32 emulation of the kernel and rejects a reference perturbed
    the ways a subtly wrong pair kernel would be: mid one row off, the h2 halo rows at an item start zeroed, b1 in place of b2,
    one row past a length left unmasked"""
    import torch
    import torch.nn.functional as F

    import tc_pair_oracle as po

    g = torch.Generator().manual_seed(3)
    C, k, dil, L, rows_item = 32, 7, 3, 700, 506
    h2 = (k - 1) // 2
    x = torch.randn(2, C, L, generator=g)
    res = torch.randn(2, C, L, generator=g)
    w1, w2 = torch.randn(C, C, k, generator=g) / (C * k) ** 0.5, torch.randn(C, C, k, generator=g) / (C * k) ** 0.5
    b1, b2 = torch.randn(C, generator=g) * 0.05, torch.randn(C, generator=g) * 0.05
    valid = [L, 400]
    ref, mid, gap = po.pair_reference(x, w1, b1, w2, b2, dil, 0.1, 0.1, res=res, res_kind="f32", valid=valid)
    bound = po.pair_bound(ref, w2, gap, valid=valid)
    mask = po.row_mask(2, L, valid, "cpu")

    def tail(m, bias=b2, mask_out=mask):
        return (F.conv1d(m, po.q16(w2.double()), bias.double(), padding=h2) + res.double()) * mask_out

    # the kernel's arithmetic: fp32 sums of the same fp16 operands
    a = po.q16(po.act32(x, 0.1)).float()
    m32 = F.conv1d(a, po.q16(w1.double()).float(), b1, padding=(k - 1) * dil // 2, dilation=dil)
    m32 = po.q16(po.lrelu(m32, 0.1) * mask.float())
    y32 = (F.conv1d(m32, po.q16(w2.double()).float(), b2, padding=h2) + res) * mask.float()
    assert po.worst_ratio(y32, ref, bound) <= 1.0

    shifted = torch.roll(mid, 1, dims=2)
    halo = mid.clone()
    halo[:, :, rows_item - h2:rows_item] = 0
    unmasked = mask.clone()
    unmasked[1, 0, 400] = 1
    for what, y in (("mid shifted one row", tail(shifted)), ("halo rows zeroed", tail(halo)), ("b1 for b2", tail(mid, b1)),
                    ("row past the length", tail(mid, mask_out=unmasked))):
        assert po.worst_ratio(y, ref, bound) > 1.0, what
