"""bench.py's reference arm (the one leg of the bench that runs without a GPU): it must print ONE JSON line with the
contract's keys, on the product arm's metric / unit / config, and never touch the CUDA library. --dump-outputs writes
the arm's last latent as float32 .npy."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]


def test_reference_arm_prints_one_contract_line(tmp_path):
    dump = tmp_path / "dump"
    out = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                          "--dump-outputs", str(dump)], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert d["impl"] == "reference"
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "e2e", "cpu_baseline"):
        assert k in d, k
    assert d["unit"] == "denoise-steps/s" and d["higher_is_better"] is True and d["steps"] == 1 and d["n_gpus"] == 1
    assert d["config"]["id"] == "c2" and "768x768" in d["config"]["workload"]
    assert d["value"] > 0 and abs(d["value"] - 1e3 / d["ms_per_step"]) < 1e-6 * d["value"] + 1e-9
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["sample"]
    e = d["e2e"]
    assert e["value"] == d["value"] and e["unit"] == d["unit"] and e["h2d_bytes_per_step"] == 0 and e["d2h_bytes_per_step"] == 0
    assert d["vs_baseline"] is None
    lat = np.load(dump / "latent.npy")
    assert lat.dtype == np.float32 and lat.ndim == 4 and lat.shape[:2] == (1, 4) and np.isfinite(lat).all()
