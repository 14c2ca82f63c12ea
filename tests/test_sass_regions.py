"""scripts/sass_regions.py: the region markers of csrc/sp_encode.cu parse into the ranges the counter needs, and the
counter runs on the built library without a GPU (when the CUDA binary tools are installed)."""
import importlib.util
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "scripts", "sass_regions.py")
SOURCE = os.path.join(ROOT, "xllm_service_b200", "csrc", "sp_encode.cu")
LIB = os.path.join(ROOT, "xllm_service_b200", "libxllm_ingest.so")


def _module():
    spec = importlib.util.spec_from_file_location("sass_regions", SCRIPT)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_markers_parse(tmp_path):
    src = tmp_path / "k.cu"
    src.write_text("a\n// region: one\nb\nc\n  // region: two (cold)\nd\n// region: end\ne\n// region: three\nf\n")
    assert _module().marker_regions(str(src)) == [("one", 2, 4, False), ("two", 5, 6, True), ("three", 9, 10, False)]


def test_express_step_is_marked():
    regions = _module().marker_regions(SOURCE)
    names = [r[0] for r in regions]
    assert len(names) == len(set(names)), names
    hot = {r[0] for r in regions if not r[3]}
    assert {"classify", "starts", "scatter-loop", "words", "key", "probe", "emit", "tail"} <= hot
    assert {"slow-classify", "miss", "blank-foreign"} <= {r[0] for r in regions if r[3]}
    assert all(first <= last for _, first, last, _ in regions)


@pytest.mark.skipif(not (shutil.which("nvdisasm") and shutil.which("cuobjdump")), reason="CUDA binary tools not on PATH")
@pytest.mark.skipif(not os.path.exists(LIB), reason="library not built")
def test_counts_the_built_library():
    out = subprocess.run([sys.executable, SCRIPT, LIB, "--weight", "scatter-loop=5"], check=True, capture_output=True,
                         text=True).stdout
    rows = {line.split()[0]: line.split() for line in out.splitlines()[2:] if line.split()}
    assert int(rows["probe"][1]) > 0 and int(rows["emit"][1]) > 0 and rows["miss"][2] == "cold"
    assert float(out.splitlines()[-1].split()[-1]) > 0
