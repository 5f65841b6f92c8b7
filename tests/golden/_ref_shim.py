"""Import the reference's own util modules from a checkout of the original Marigold repository (path in
$MARIGOLD_REFERENCE) WITHOUT importing `marigold/__init__` (which needs diffusers). Used by make_golden.py to produce
the committed fixtures; the tests never need it. matplotlib is stubbed (only colorize_depth_maps uses it)."""
import importlib.util
import os
import sys
import types
from pathlib import Path

REF = Path(os.environ.get("MARIGOLD_REFERENCE", "reference"))


def load_reference_utils():
    if not (REF / "marigold" / "util").is_dir():
        raise RuntimeError(f"no Marigold checkout at {REF} (set MARIGOLD_REFERENCE to regenerate the fixtures)")
    if "matplotlib" not in sys.modules:
        sys.modules["matplotlib"] = types.ModuleType("matplotlib")
    pkg = types.ModuleType("refmarigold")
    pkg.__path__ = [str(REF / "marigold")]
    sys.modules["refmarigold"] = pkg
    util = types.ModuleType("refmarigold.util")
    util.__path__ = [str(REF / "marigold" / "util")]
    sys.modules["refmarigold.util"] = util
    mods = {}
    for name in ("image_util", "ensemble", "batchsize"):
        spec = importlib.util.spec_from_file_location(f"refmarigold.util.{name}", REF / "marigold" / "util" / f"{name}.py")
        m = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = m
        spec.loader.exec_module(m)
        mods[name] = m
    return mods
