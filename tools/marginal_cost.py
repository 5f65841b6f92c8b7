"""In-graph marginal cost of each kernel family: step time with the family removed (MGB_SKIP) vs full."""
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
res = {}
for fam in ["", "gn", "ln", "attn", "xattn", "gemm", "gn,ln,attn,xattn", "gn,ln,attn,xattn,gemm"]:
    env = dict(os.environ)
    if fam:
        env["MGB_SKIP"] = fam
    out = subprocess.run([sys.executable, str(ROOT / "tools" / "step_only.py"), "12"], env=env, capture_output=True, text=True)
    line = [l for l in out.stdout.splitlines() if "ms/step" in l]
    ms = float(line[-1].split("steps:")[1].split("ms/step")[0]) if line else None
    res[fam or "full"] = ms
    print(fam or "full", ms, flush=True)
full = res["full"]
print(json.dumps({k: (None if v is None else round(full - v, 3)) for k, v in res.items()}))
(ROOT / "out").mkdir(exist_ok=True)
(ROOT / "out" / "marginal_cost.json").write_text(json.dumps(res, indent=1))
