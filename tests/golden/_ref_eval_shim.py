"""Import the reference's evaluation helpers, src/util/metric.py (needs pandas) and src/util/alignment.py, from a checkout
of the original Marigold repository (path in $MARIGOLD_REFERENCE, as for _ref_shim.py) without importing the `src`
package, whose __init__ pulls in the training stack. Used by make_eval_golden.py; the tests never need it."""
import importlib.util
import sys

from tests.golden._ref_shim import REF


def load_reference_eval_utils():
    if not (REF / "src" / "util").is_dir():
        raise RuntimeError(f"no Marigold checkout at {REF} (set MARIGOLD_REFERENCE to regenerate the fixtures)")
    mods = {}
    for name in ("metric", "alignment"):
        spec = importlib.util.spec_from_file_location(f"refsrc_util_{name}", REF / "src" / "util" / f"{name}.py")
        m = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = m
        spec.loader.exec_module(m)
        mods[name] = m
    return mods
