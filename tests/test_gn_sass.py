"""The persistent kernel's item loop touches no local memory at any shape the automatic choice may pick.

A spill inside k_gn_loop's item loop is paid once per (moving leaf, keyframe) pair in every round, and it is what made the
larger shapes slow per pass; pick_shape only considers the shapes of madicp_ctx::kAutoShapes (ctx.hpp).  The loop and the
rule (save / restore around the out-of-line exact side test and the sqrt / reciprocal slow paths do not count) are
defined in scripts/sass_census.py.  Needs cuobjdump (CUDA toolkit); no GPU."""
import importlib.util
import os
import re
import shutil

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUOBJDUMP = shutil.which("cuobjdump") or next(
    (p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.access(p, os.X_OK)), None)
pytestmark = pytest.mark.skipif(CUOBJDUMP is None, reason="cuobjdump not found")


def _census():
    spec = importlib.util.spec_from_file_location("sass_census", os.path.join(ROOT, "scripts", "sass_census.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _auto_shapes():
    src = open(os.path.join(ROOT, "mad_icp_b200", "csrc", "ctx.hpp")).read()
    m = re.search(r"kAutoShapes\[kNumAutoShapes\]\s*=\s*\{([^}]*)\}", src)
    return [int(v) for v in m.group(1).split(",")]


@pytest.fixture(scope="module")
def sass():
    census = _census()
    assert os.path.exists(census.LIB), "build the library first"
    return census, census.sass(tool=CUOBJDUMP)


def test_auto_shapes_have_no_local_memory_in_item_loop(sass):
    census, txt = sass
    shapes = _auto_shapes()
    assert shapes and set(shapes) <= set(census.SHAPES)
    for t in shapes:
        counted, _ = census.item_loop_local_ops(census.kernel_body(txt, t))
        assert not counted, f"k_gn_loop<{t},1>: " + ", ".join(f"{op} at {a:#x}" for a, op in counted)


def test_item_loop_holds_the_fold_and_the_walk(sass):
    # the loop the census judges is the item loop: it holds the 8 DMMA of the fold and the walk's 128-bit loads
    census, txt = sass
    for t in census.SHAPES:
        ins = census.instructions(census.kernel_body(txt, t))
        lo, hi = census.item_loop_range(ins)
        inside = [op for a, op, _ in ins if lo <= a <= hi]
        assert sum(op.startswith("DMMA") for op in inside) == 8, t
        assert sum(op.startswith("LDG.E.128.CONSTANT") for op in inside) >= 4, t
