"""The f16tc path has run-time switches for A/B measurements (MB_TC_FUSE, MB_TC_RES16, MB_TC_X3_RES16, MB_TC_RED_ADD, MB_TC_SPLIT3,
MB_TC_UPS_X3, MB_POST_TILE, MB_POST_ROWS; read once per process).  Every combination a user can select must stay inside the 1e-3
tolerance: each setting runs the golden comparison in a fresh interpreter."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent

SCRIPT = r"""
import json, sys
sys.path.insert(0, "oracle"); sys.path.insert(0, "synth_weights")
import numpy as np, torch
import gan_oracle as go, ref_init as ri
from mockingbird_b200.vocoder.hifigan.models import Generator
cfg = ri.HIFIGAN_CONFIG_16K
g = Generator(cfg, precision="f16tc").cuda()
g.load_state_dict(ri.hifigan_state_dict(cfg, 0)); g.eval(); g.remove_weight_norm()
z = np.load("tests/golden/hifigan_seed0.npz")
out = {}
wav = g(torch.from_numpy(z["mel_small"]).cuda()).cpu()
out["small"] = go.rel_errors(wav, torch.from_numpy(z["wav_small"]))
mel = torch.rand(3, 80, 70, generator=torch.Generator().manual_seed(5)) * 8 - 4
lens = torch.tensor([70, 33, 1], dtype=torch.int32)
wav = g(mel.cuda(), lengths=lens.cuda()).cpu()
sd = go.fold_weight_norm(ri.hifigan_state_dict(cfg, 0))
worst = 0.0
tail = 0.0
for b in range(3):
    t = int(lens[b])
    ref = go.hifigan_forward(sd, cfg, mel[b:b + 1, :, :t])
    e = go.rel_errors(wav[b:b + 1, :, : t * 200], ref)
    worst = max(worst, e["max_rel"], e["rms_rel"])
    if t < 70:
        tail = max(tail, float(wav[b, :, t * 200:].abs().max()))
out["ragged_worst"] = worst
out["tail"] = tail
print(json.dumps(out))
"""

ENVS = [{}, {"MB_TC_UPS_X3": "0", "MB_TC_RES16": "0"}, {"MB_TC_FUSE": "0"}, {"MB_TC_RES16": "0", "MB_TC_FUSE": "0"}, {"MB_TC_UPS_X3": "0"}, {"MB_TC_RES16": "0"}, {"MB_TC_X3_RES16": "0"},
        {"MB_POST_ROWS": "1"}, {"MB_POST_ROWS": "4"}, {"MB_TC_RED_ADD": "0"}, {"MB_POST_TILE": "1"}, {"MB_TC_SPLIT3": "0"},
        {"MB_TC_RES16": "0", "MB_TC_RED_ADD": "0", "MB_TC_SPLIT3": "0"}]


@pytest.mark.parametrize("env", ENVS, ids=lambda e: ",".join(f"{k}={v}" for k, v in e.items()) or "default")
def test_hifigan_f16tc_switches_within_tolerance(env):
    e = dict(os.environ)
    e.update(env)
    r = subprocess.run([sys.executable, "-c", SCRIPT], cwd=ROOT, env=e, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["small"]["max_rel"] <= 1e-3 and out["small"]["rms_rel"] <= 1e-3, out
    assert out["ragged_worst"] <= 1e-3, out
    assert out["tail"] == 0.0, out  # samples past an utterance's length are exactly zero
