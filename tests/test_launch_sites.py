"""CPU: every kernel of libb200gp.so is launched through common.cuh's launch() / count_launch().

Those two check the launch where it is made and count it in ctx->launches, whose difference over a call is
b2gp_timing::launches (bench.py's gpu_launches).  A launch written out anywhere else would be counted by hand or not at
all.  The kernel path counters are kept there too; only the three route counters are bumped by count_path() at the
entry of their route."""
import pathlib
import re

CSRC = pathlib.Path(__file__).resolve().parents[1] / "gpax_b200" / "csrc"
ROUTES = {"PATH_PANEL_SOLVE", "PATH_TRSM_TALL", "PATH_POTRF_TALL"}
KERNEL_COUNTERS = {"PATH_GEMM_NT", "PATH_GEMM_TMA", "PATH_OZ_MMA", "PATH_OZ_SLICE", "PATH_TRSM_STRIP", "PATH_POTRF_DIAG"}
LAUNCH_COUNT_WRITE = re.compile(r"ctx->launches\s*(\+\+|--|[-+]?=(?!=))|(\+\+|--)\s*ctx->launches\b")
# the helpers in common.cuh: function definitions that end at a closing brace in column 0
HELPER = re.compile(r"^(?:template <[^\n]*>\n)?static (?:inline )?int (?:count_launch|launch)\(.*?^}\n", re.S | re.M)


def code(path):
    """the source without comments"""
    text = re.sub(r"/\*.*?\*/", "", path.read_text(), flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def sources():
    files = {p.name: code(p) for p in sorted(CSRC.iterdir()) if p.suffix in (".cu", ".cuh")}
    assert "common.cuh" in files and "b200gp.cu" in files
    return files


def split_helpers(files):
    """(the text of common.cuh's launch helpers, every source with those helpers cut out)"""
    helpers = HELPER.findall(files["common.cuh"])
    assert len(helpers) == 3, "count_launch and the two launch() overloads"
    rest = dict(files, **{"common.cuh": HELPER.sub("", files["common.cuh"])})
    return "".join(helpers), rest


def test_kernels_are_launched_and_counted_only_by_the_helpers():
    helpers, rest = split_helpers(sources())
    assert helpers.count("<<<") == 1 and len(LAUNCH_COUNT_WRITE.findall(helpers)) == 1
    for name, text in rest.items():
        for i, line in enumerate(text.splitlines(), 1):
            assert "<<<" not in line, f"{name}:{i}: kernel launched outside launch(): {line.strip()}"
            assert not LAUNCH_COUNT_WRITE.search(line), f"{name}:{i}: ctx->launches written outside count_launch(): {line.strip()}"


def test_count_path_outside_the_helpers_names_only_route_counters():
    _, rest = split_helpers(sources())
    named = {m for text in rest.values() for m in re.findall(r"\bcount_path\(\s*ctx\s*,\s*(\w+)\s*\)", text)}
    assert named <= ROUTES, f"kernel counters bumped by hand: {sorted(named - ROUTES)}"
    assert named == ROUTES, f"route counters no longer counted: {sorted(ROUTES - named)}"
    launched = {m for text in rest.values() for m in re.findall(r"\b(?:launch|count_launch)\(\s*ctx\s*,\s*(PATH_\w+)", text)}
    assert launched == KERNEL_COUNTERS
