"""GPU bring-up battery for the hand-written kernels: every case compares a C-ABI operator call with a
plain torch fp32 computation on the same bf16-rounded inputs, and reports max error + a CUDA-event
timing. Cases run in a child process; a trap / hang in one case is recorded and the battery resumes
with the next case in a fresh process (a trapped context is unusable).

    python tools/bringup.py --all [--filter gemm] [--out out/bringup.jsonl]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


from tests.ops_cases import cases as _cases  # noqa: E402


# -------------------------------------------------------------------------------------------------
def child(start, flt, out_path):
    import torch

    cases = [c for c in _cases() if (flt is None or flt in c[0])]
    assert torch.cuda.is_available(), "bring-up needs a GPU"
    from marigold_b200 import _lib

    _lib.load()
    with open(out_path, "a") as f:
        for i in range(start, len(cases)):
            name, fn, kw = cases[i]
            f.write(json.dumps({"case": name, "index": i, "status": "started"}) + "\n")
            f.flush()
            os.fsync(f.fileno())
            t0 = time.time()
            try:
                res = fn(**kw)
                torch.cuda.synchronize()
                rec = {"case": name, "index": i, "status": "done", "wall_s": round(time.time() - t0, 3), **res}
            except Exception as e:  # noqa: BLE001
                rec = {"case": name, "index": i, "status": "error", "error": repr(e)[:500]}
                f.write(json.dumps(rec) + "\n")
                f.flush()
                print(json.dumps(rec), flush=True)
                if "CUDA" in repr(e) or "cuda" in repr(e):
                    return 17  # context is probably dead: let the parent restart after this case
                continue
            f.write(json.dumps(rec) + "\n")
            f.flush()
            print(json.dumps(rec), flush=True)
    return 0


def parent(flt, out_path, per_child_timeout):
    n = len([c for c in _cases() if (flt is None or flt in c[0])])
    Path(out_path).parent.mkdir(parents=True, exist_ok=True)
    Path(out_path).write_text("")
    start = 0
    while start < n:
        cmd = [sys.executable, __file__, "--child", str(start), "--out", out_path]
        if flt:
            cmd += ["--filter", flt]
        try:
            r = subprocess.run(cmd, timeout=per_child_timeout)
            rc = r.returncode
        except subprocess.TimeoutExpired:
            rc = -9
        # find the last started/done index
        last_started, last_done = -1, -1
        for line in Path(out_path).read_text().splitlines():
            rec = json.loads(line)
            if rec["status"] == "started":
                last_started = rec["index"]
            else:
                last_done = rec["index"]
        if rc == 0 and last_done >= n - 1:
            break
        if last_started > last_done:
            with open(out_path, "a") as f:
                f.write(json.dumps({"case": "?", "index": last_started, "status": "crashed", "rc": rc}) + "\n")
            print(json.dumps({"index": last_started, "status": "crashed", "rc": rc}), flush=True)
        start = max(last_started, last_done) + 1
    # summary
    recs = {}
    names = {}
    for line in Path(out_path).read_text().splitlines():
        rec = json.loads(line)
        if rec["status"] == "started":
            names[rec["index"]] = rec["case"]
        else:
            recs[rec["index"]] = rec
    bad = []
    for i in range(n):
        rec = recs.get(i, {"status": "missing"})
        ok = rec.get("status") == "done" and rec.get("ok", False)
        if not ok:
            bad.append(names.get(i, str(i)))
    print(f"BRINGUP SUMMARY: {n - len(bad)}/{n} ok; failing: {bad}", flush=True)
    return 0 if not bad else 1


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--all", action="store_true")
    ap.add_argument("--child", type=int, default=None)
    ap.add_argument("--filter", default=None)
    ap.add_argument("--out", default=str(ROOT / "out" / "bringup.jsonl"))
    ap.add_argument("--timeout", type=int, default=240)
    a = ap.parse_args()
    if a.child is not None:
        sys.exit(child(a.child, a.filter, a.out))
    sys.exit(parent(a.filter, a.out, a.timeout))
