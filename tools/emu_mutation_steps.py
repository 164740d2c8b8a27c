"""Mutation check of the captured step's kernels (tests/emu_fuzz.py: fuzz_graphed_step).

Each mutant changes ONE piece of the code a GraphedContrastStep replay runs — the dense-gradient scatter into sectors
(k_scatter_reduce), the sparse-reset clear in k_select and the record it reads, the live tile counts of the one-kernel
InfoNCE (k_self_fused), the step's zero-fill and the plane fill of k_zero_scatter — in a scratch copy of the sources,
built for the emulator.  Two suites run against every mutant:

  old  the emulated tests that reached these kernels before the graphed-step fuzzer was extended: test_emu_kernels.py,
       test_emu_mixed_precision.py and test_emu_fuzz.py with the fuzzer of commit OLD_REV (read from git)
  new  test_emu_fuzz.py::test_fuzz_graphed_step

A suite kills a mutant when a test fails or the process aborts.  Nothing in the tree is modified.

Three mutants the check started from are EQUIVALENT (no test can kill them) and run as a control, expected to survive:
  * skip rule r < s -> r > s: one anchor of a shared sector writes every value in it, so it does not matter which one;
  * prev_rows[0] = max_samples instead of A: the extra rows are clears of entries an earlier replay already cleared,
    and every clear runs before the scatter of its replay;
  * k_self_fused's live tiles from a_rows instead of A: the kernel also masks rows and columns at A (valid, jend), so
    the tiles past A add zeros — the mutant costs time, not values.
Their non-equivalent neighbours (r != s: a shared sector is never written; A - 1: a row is never cleared; negatives up
to a_rows: the zero rows past A count as negatives) are in the list.  The emulator runs the one-kernel InfoNCE one phase per launch and the fill branch inline: mutants of the inter-CTA
barriers or of the fill-versus-scatter order need real concurrency, and the device fuzzer
(tests/test_gpu_sm_regimes.py::test_fuzz_captured_steps_on_the_device) is their check.

    python tools/emu_mutation_steps.py      # one line per mutant; exit 1 if a mutant survives the new suite
"""
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import build_emu as b  # noqa: E402

OLD_REV = "8c08ac2"          # the last commit with the eager-only graphed-step fuzzer
SEL, STEP, FUSED = "pcl_select.cu", "pcl_step.cu", "pcl_infonce_fused.cu"
MUTANTS = [   # (name, source file, exact text, replacement, equivalent)
    ("k_scatter_reduce: no clamp of the splits to the live column tiles", SEL,
     "if (split_cols > 0) src.splits = min(src.splits, (A + split_cols - 1) / split_cols);", "", False),
    ("sector skip rule r < s -> r > s (the highest anchor writes the sector)", SEL,
     "if (r < s) s_skip = 1;", "if (r > s) s_skip = 1;", True),
    ("sector skip rule r < s -> r != s (a shared sector is never written)", SEL,
     "if (r < s) s_skip = 1;", "if (r != s) s_skip = 1;", False),
    ("sector path: the value of anchor s in every owned element", SEL,
     "src.at(own, d, D, scale)", "src.at(s, d, D, scale)", False),
    ("prev_rows[0] = max_samples instead of A", SEL,
     "prev_rows[0] = A;", "prev_rows[0] = g.max_samples;", True),
    ("prev_rows[0] = A - 1 (the last row of a replay is never cleared)", SEL,
     "prev_rows[0] = A;", "prev_rows[0] = A - 1;", False),
    ("k_select: sparse clear of one row less", SEL,
     "if (ip < min(prev_rows[0], msp)) {", "if (ip < min(prev_rows[0], msp) - 1) {", False),
    ("k_self_fused: live tiles from a_rows instead of A", FUSED,
     "const int R_live = (A + BM - 1) / BM, S_live = (A + BN - 1) / BN;",
     "const int R_live = (a.a_rows + BM - 1) / BM, S_live = (a.a_rows + BN - 1) / BN;", True),
    ("k_self_fused: negatives up to a_rows instead of A (the dead rows count as negatives)", FUSED,
     "jend[h] = valid ? A - col0 : 0;", "jend[h] = valid ? a.a_rows - col0 : 0;", False),
    ("pcl_step_fused_fill: element size fixed at 2", STEP,
     "d->g.h * d->g.w * pcl::dtype_size(d->embed_dtype);", "d->g.h * d->g.w * 2;", False),
    ("zero_plane: the 16-byte branch stores HW / E - 1 vectors", SEL,
     "i < HW / E; i += blockDim.x) d4[i] = z;", "i < HW / E - 1; i += blockDim.x) d4[i] = z;", False),
]
NEW_SUITE = ["tests/test_emu_fuzz.py::test_fuzz_graphed_step"]


def old_suite(tmp):
    """The parent's fuzzer and its test file in `tmp` (imported before the tree's)."""
    for name in ("emu_fuzz.py", "test_emu_fuzz.py"):
        text = subprocess.run(["git", "show", f"{OLD_REV}:tests/{name}"], cwd=ROOT, capture_output=True, text=True,
                              check=True).stdout
        with open(os.path.join(tmp, name), "w") as f:
            f.write(text)
    return [os.path.join(tmp, "test_emu_fuzz.py"), "tests/test_emu_kernels.py", "tests/test_emu_mixed_precision.py"]


def build_mutant(i, fname, old, new):
    out = f"/tmp/pcl_emu_steps_mutant_{i}"
    os.makedirs(out, exist_ok=True)
    cpps = []
    for name in b.SOURCES:
        text = open(os.path.join(b.CSRC, name)).read()
        if name == fname:
            assert text.count(old) == 1, f"mutant {i}: source text not found once: {old}"
            text = text.replace(old, new)
        p = os.path.join(out, name[:-3] + ".emu.cpp")
        with open(p, "w") as f:
            f.write(b.rewrite(text))
        cpps.append(p)
    cpps.append(os.path.join(b.HERE, "emu_tc_stubs.cpp"))
    lib = os.path.join(out, "libpcl_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-ffp-contract=off", "-fno-strict-aliasing", "-w",
                    "-Wno-psabi", "-DPCL_EMU_SMS=6", "-I", os.path.join(b.HERE, "shim"), "-I", b.CSRC, "-I",
                    os.path.join(b.ROOT, "include"), "-x", "c++"] + cpps + ["-o", lib], check=True)
    return lib


def run_suite(lib, args, first=None):
    pre = (f"sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})\nsys.path.insert(0, {first!r})\nimport emu_fuzz\n"
           if first else "")
    code = (f"import sys\nsys.path.insert(0, {os.path.join(ROOT, 'tests', 'emu')!r})\nimport build_emu\n"
            f"build_emu.build = lambda force=False, sms=6: {lib!r}\n{pre}import pytest\n"
            f"sys.exit(pytest.main({args + ['-q', '-x', '-p', 'no:cacheprovider', '-m', 'not gpu']!r}))\n")
    return subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=7200).returncode


def check(i, tmp, old_args):
    name, fname, old, new, equivalent = MUTANTS[i]
    lib = build_mutant(i, fname, old, new)
    rc_old, rc_new = run_suite(lib, old_args, first=tmp), run_suite(lib, NEW_SUITE)
    how = lambda rc: "abort" if rc < 0 else ("killed" if rc else "survived")     # noqa: E731
    return name, how(rc_old), how(rc_new), equivalent


if __name__ == "__main__":
    with tempfile.TemporaryDirectory() as tmp:
        old_args = old_suite(tmp)
        with ThreadPoolExecutor(min(len(MUTANTS), max(1, (os.cpu_count() or 2) // 2))) as ex:
            res = list(ex.map(lambda i: check(i, tmp, old_args), range(len(MUTANTS))))
    for name, old, new, eq in res:
        print(f"old suite: {old:8s}  new suite: {new:8s}  {name}{'  (equivalent: control)' if eq else ''}", flush=True)
    sys.exit(1 if any(new == "survived" and not eq for _, _, new, eq in res) else 0)
