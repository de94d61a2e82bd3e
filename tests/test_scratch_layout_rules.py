"""Every batched call (blockIdx.y = job) lays out its device scratch through one helper, Layout in common.cuh: the same layout code
runs once to measure and once to place, so the size a buffer is ensured to and the regions placed in it cannot disagree.  The
batched scan's tile state (its size, the tile counter behind the tile words) is known to runtime.cu alone: callers take each job's
state through scan_bind_state.  These tests read the CUDA sources and fail when a source rounds its own regions or computes a scan
state again.  No GPU needed."""
import glob
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "open3d_slam_b200", "csrc")
SOURCES = sorted(os.path.basename(p) for p in glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")))
ROUND_256 = re.compile(r"\((\w+) \+ 255\) & ~\(size_t\)255")


def source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_one_layout_rounding():
    for name in SOURCES:
        src = source(name)
        found = ROUND_256.findall(src)
        if name == "common.cuh":
            assert found == ["bytes"], f"common.cuh: {found}"
            layout = re.search(r"struct Layout \{(.*?)\n\};", src, re.S)
            assert layout and ROUND_256.search(layout.group(1)), "the 256-byte rounding belongs to Layout"
        elif name == "runtime.cu":
            assert found == ["ncap"], f"runtime.cu: only DevBuf::ensure's capacity rounding may stay, found {found}"
        else:
            assert not found, f"{name}: own 256-byte rounding {found}"
        assert not re.search(r"\+ 15\) & ~\(size_t\)15", src), f"{name}: own 16-byte rounding"
        for helper in (r"auto al\b", r"\bal256\b", r"static inline size_t al\b"):
            assert not re.search(helper, src), f"{name}: own alignment helper ({helper})"


def test_scan_state_known_to_runtime_only():
    for name in SOURCES:
        if name in ("runtime.cu", "common.cuh"):
            continue
        src = source(name)
        assert "scan_state_bytes(" not in src, f"{name}: sizes a scan tile state itself"
        assert "- 64) / 8" not in src, f"{name}: locates a scan tile counter itself"


def test_overlap_stage_size_gone():
    for name in SOURCES:
        assert "op_overlap_batch_stage_bytes" not in source(name), name


def test_batched_scans_bind_their_states():
    callers = [n for n in SOURCES if n not in ("runtime.cu", "common.cuh") and "scan_exclusive_i32_batch(" in source(n)]
    assert len(callers) >= 5, callers
    for name in callers:
        src = source(name)
        assert "scan_bind_state(" in src, f"{name}: runs the batched scan without scan_bind_state"
        assert not re.search(r"\.(state|counter)\s*=[^=]", src), f"{name}: sets a ScanJob's state or counter itself"
