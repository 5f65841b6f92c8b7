"""Generate tests/golden/*.npz by running the REFERENCE's own functions (needs a checkout of the original
Marigold repository, path in $MARIGOLD_REFERENCE). Inputs are regenerated from seeds by tests/golden/cases.py, so only the
reference outputs are stored.

    python tests/golden/make_golden.py
"""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from tests.golden._ref_shim import load_reference_utils  # noqa: E402
from tests.golden.cases import (DEPTH_CASES, IID_CASES, NORMALS_CASES, RESIZE_CASES, depth_input, iid_input,  # noqa: E402
                                normals_input, resize_input)

ref = load_reference_utils()
out_dir = Path(__file__).resolve().parent
torch.set_num_threads(4)

import scipy.optimize as so  # noqa: E402

_orig_min = so.minimize
_last = {}


def _spy(*a, **k):
    r = _orig_min(*a, **k)
    _last.update(x0=np.array(a[1], dtype=np.float64), x=np.array(r.x, dtype=np.float64), nit=r.nit, nfev=r.nfev)
    return r


so.minimize = _spy
import scipy  # noqa: E402

scipy.optimize.minimize = _spy

# ensemble_iid (marigold/util/ensemble.py:250-270): a separate small file so that the depth / normals goldens stay
# byte-identical
iid = {}
for name, cfg in IID_CASES.items():
    pred, unc = ref["ensemble"].ensemble_iid(iid_input(cfg).clone(), **dict(cfg.get("kwargs", {})))
    iid[f"iid/{name}/pred"] = pred.numpy()
    if unc is not None:
        iid[f"iid/{name}/unc"] = unc.numpy()
np.savez_compressed(out_dir / "iid_golden.npz", **iid)
print("iid cases", sorted(iid))
if "--iid-only" in sys.argv:
    sys.exit(0)

store = {}
for name, cfg in DEPTH_CASES.items():
    d = depth_input(cfg)
    kw = dict(cfg.get("kwargs", {}))
    _last.clear()
    pred, unc = ref["ensemble"].ensemble_depth(d.clone(), **kw)
    store[f"depth/{name}/pred"] = pred.numpy()
    if unc is not None:
        store[f"depth/{name}/unc"] = unc.numpy()
    if _last:
        store[f"depth/{name}/x0"] = _last["x0"]
        store[f"depth/{name}/x"] = _last["x"]
        store[f"depth/{name}/nit"] = np.array(_last["nit"])
        store[f"depth/{name}/nfev"] = np.array(_last["nfev"])
    print(name, "nit", _last.get("nit"), "nfev", _last.get("nfev"), "moved",
          float(np.abs(_last["x"] - _last["x0"]).max()) if _last else None)
for name, cfg in NORMALS_CASES.items():
    n = normals_input(cfg)
    kw = dict(cfg.get("kwargs", {}))
    pred, unc = ref["ensemble"].ensemble_normals(n.clone(), **kw)
    store[f"normals/{name}/pred"] = pred.numpy()
    if unc is not None:
        store[f"normals/{name}/unc"] = unc.numpy()
    # the index the reference's argmax picked (recomputed with the reference's exact expressions)
    mean_n = n.mean(dim=0, keepdim=True)
    mean_n = mean_n / torch.norm(mean_n, dim=1, keepdim=True).clamp(min=1e-6)
    sim = (mean_n * n).sum(dim=1, keepdim=True).clamp(-1, 1)
    store[f"normals/{name}/argmax"] = sim.argmax(dim=0, keepdim=True).numpy().astype(np.int32)
try:
    from torchvision.transforms import InterpolationMode  # noqa: F401

    for name, cfg in RESIZE_CASES.items():
        img = resize_input(cfg)
        m = ref["image_util"].get_tv_resample_method(cfg["method"])
        store[f"resize/{name}"] = ref["image_util"].resize_max_res(img, cfg["max_edge"], m).numpy()
except Exception as e:  # noqa: BLE001
    print("resize goldens skipped:", e)
np.savez_compressed(out_dir / "ensemble_golden.npz", **store)
print("wrote", out_dir / "ensemble_golden.npz", sum(v.nbytes for v in store.values()) / 1e6, "MB raw")
