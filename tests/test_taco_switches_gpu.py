"""Every run-time switch of the Tacotron and speaker-encoder paths (DESIGN.md section 6b), one fresh interpreter per setting (the
switches are read once per process).  Each setting runs Tacotron golden `a`, a B = 70 oracle case (65-127 rows: the second MMA
warpgroup with a partial row range) and the encoder goldens, within the existing tolerances.

MB_TACO_GRAPH, MB_TACO_PDL, MB_TACO_PDL2, MB_TACO_RING8 and MB_TACO_MC change only how the same kernels are scheduled: graph
replay vs direct launches, programmatic dependent launch, the ring depth of the compact activation slots, multicast of the
same activation bytes.  No product or sum changes order, so their outputs must equal the default's bit for bit."""
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import ref_init as ri
import tacotron_oracle as to

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
TACO_TOL, ENC_TOL = 2e-4, 1e-4

SCRIPT = r"""
import sys
sys.path.insert(0, "oracle"); sys.path.insert(0, "synth_weights")
import numpy as np, torch
import ref_init as ri
from mockingbird_b200.synthesizer.inference import Synthesizer
from mockingbird_b200.encoder import inference as enc_inf
from mockingbird_b200.encoder.model import SpeakerEncoder
out_path, case_path = sys.argv[1], sys.argv[2]
model = Synthesizer("unused.pt", verbose=False).load_state(ri.tacotron_state_dict(0, r=2, randomize_bn=True))
z = np.load("tests/golden/tacotron_seed0.npz")
enc = torch.from_numpy(np.unpackbits(z["a_enc_masks"], axis=-1))
dec = np.unpackbits(z["a_dec_masks"], axis=-1)
dec = torch.from_numpy(dec.reshape(-1, 2, dec.shape[-2], dec.shape[-1]))
steps, style, mst, r = [int(v) for v in z["a_cfg"]]
res = {}
mel, lin, attn = model.generate(torch.from_numpy(z["a_chars"]), torch.from_numpy(z["a_emb"]), steps=steps, style_idx=style,
                                min_stop_token=mst, dropout_masks=(enc, dec))
res.update(a_mel=mel.cpu().numpy(), a_linear=lin.cpu().numpy(), a_attn=attn.cpu().numpy())
c = np.load(case_path)
mel, lin, attn = model.generate(torch.from_numpy(c["chars"]), torch.from_numpy(c["emb"]), steps=int(c["steps"]), style_idx=-1,
                                min_stop_token=10, dropout_masks=(torch.from_numpy(c["enc"]), torch.from_numpy(c["dec"])))
res.update(b70_mel=mel.cpu().numpy(), b70_linear=lin.cpu().numpy(), b70_attn=attn.cpu().numpy())
m = SpeakerEncoder(); m.load_state_dict(ri.encoder_state_dict(0)); m.eval(); enc_inf.set_model(m)
ze = np.load("tests/golden/encoder_seed0.npz")
for n in ("a", "b"):
    res[f"enc_{n}"] = enc_inf.embed_frames_batch(ze[f"{n}_frames"])
np.savez(out_path, **res)
print("ok")
"""

SETTINGS = ([{f"MB_TACO_{k}": "0"} for k in ("TC", "CONV_TC", "GRAPH", "PDL", "PDL2", "PRENET_FUSED", "SPLIT_FUSED", "LSA_FUSED",
                                            "STOP_FUSED", "RING8", "DAG")]
            + [{"MB_TACO_MC": v} for v in ("2", "4", "8")] + [{"MB_ENC_TC": "0"}])
SCHEDULING_ONLY = {"MB_TACO_GRAPH", "MB_TACO_PDL", "MB_TACO_PDL2", "MB_TACO_RING8", "MB_TACO_MC"}


@pytest.fixture(scope="module")
def case(tmp_path_factory):
    """B = 70 rows, 20 chars, 12 steps, with its float32 CPU oracle result"""
    g = torch.Generator().manual_seed(7070)
    B, Tc, steps = 70, 20, 12
    chars = torch.randint(2, 75, (B, Tc), generator=g)
    for b in range(0, B, 4):
        chars[b, 6 + (b % 9):] = 0
    emb = torch.rand(B, 256, generator=g)
    emb = emb / emb.norm(dim=1, keepdim=True)
    enc = torch.rand(2, B, Tc, 256, generator=g) < 0.5
    dec = torch.rand(steps // 2, 2, B, 256, generator=g) < 0.5
    masks = [enc[0], enc[1]] + [dec[i, j] for i in range(steps // 2) for j in range(2)]
    sd = ri.tacotron_state_dict(0, r=2, randomize_bn=True)
    mel, lin, attn = to.generate(sd, chars, emb, steps, -1, 10, masks, r=2)
    p = tmp_path_factory.mktemp("taco_switch") / "case.npz"
    np.savez(p, chars=chars.numpy(), emb=emb.numpy(), enc=enc.numpy(), dec=dec.numpy(), steps=steps)
    return p, {"mel": mel.numpy(), "linear": lin.numpy(), "attn": attn.numpy()}


def _run(env, case_path, out):
    e = dict(os.environ)
    e.update(env)
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(out), str(case_path)], cwd=ROOT, env=e, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return dict(np.load(out))


@pytest.fixture(scope="module")
def default(case, tmp_path_factory):
    return _run({}, case[0], tmp_path_factory.mktemp("taco_switch") / "default.npz")


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def _check_tolerances(got, case, golden_dir):
    z = np.load(golden_dir / "tacotron_seed0.npz")
    for key in ("mel", "linear", "attn"):
        assert got[f"a_{key}"].shape == z[f"a_{key}"].shape, key
        assert _rel(got[f"a_{key}"], z[f"a_{key}"]) <= TACO_TOL, ("a", key, _rel(got[f"a_{key}"], z[f"a_{key}"]))
        ref = case[1][key]
        assert got[f"b70_{key}"].shape == ref.shape, key
        assert _rel(got[f"b70_{key}"], ref) <= TACO_TOL, ("b70", key, _rel(got[f"b70_{key}"], ref))
    ze = np.load(golden_dir / "encoder_seed0.npz")
    for n in ("a", "b"):
        assert np.abs(got[f"enc_{n}"] - ze[f"{n}_embeds"]).max() < ENC_TOL, n


def test_default_within_tolerance(default, case, golden_dir):
    _check_tolerances(default, case, golden_dir)


@pytest.mark.parametrize("env", SETTINGS, ids=lambda e: ",".join(f"{k}={v}" for k, v in e.items()))
def test_switch(env, default, case, golden_dir, tmp_path):
    got = _run(env, case[0], tmp_path / "out.npz")
    _check_tolerances(got, case, golden_dir)
    same = {k: bool(np.array_equal(got[k], default[k])) for k in default}
    print(json.dumps({"env": env, "bitwise_equal": same}))
    if set(env) & SCHEDULING_ONLY:
        assert all(same.values()), same
