"""Mutation check of the work splits that depend on the SM count (tests/test_emu_sm_counts.py).

Each mutant changes ONE piece of the arithmetic that sizes a grid, a work list or a partial-sum workspace from the SM
count, in a scratch copy of the sources.  It is built for the emulator at 6 SMs (the count of the rest of the emulated
suite) and at 7, 114 and 132 SMs, then run against two suites: the emulated tests that reach these kernels at 6 SMs,
and tests/test_emu_sm_counts.py.  A suite kills a mutant when a test fails or the process aborts.  Nothing in the tree
is modified.

    python tools/emu_mutation_sms.py        # one line per mutant; exit 1 if a mutant survives the new tests
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import build_emu as b  # noqa: E402

TC, NORM = "pcl_infonce_tc.cu", "pcl_norm.cu"
MUTANTS = [   # (name, source file, exact text, replacement)
    ("k_tc_fwd: no clamp of the grid to the live pairs", TC, "if (w0.G > w0.P) w0.G = (int)w0.P;", ""),
    ("neg_slot_bound: without the + 2 (host slots and POS prologues)", TC, "col_tiles / (U > 1 ? U : 1) + 2;",
     "col_tiles / (U > 1 ? U : 1);"),
    ("make_tc_plan: splits not capped by col_tiles", TC, "  if (splits > col_tiles) splits = col_tiles;\n", ""),
    ("layout(): ctiles from Cin instead of Cin + 1", NORM, "L.ctiles = ceil_div(Cin + 1, DOUT);",
     "L.ctiles = ceil_div(Cin, DOUT);"),
    ("k_tc_pos_t: units per CTA rounded down (last units dropped)", TC,
     "int U = (P + (int)gridDim.x - 1) / (int)gridDim.x;", "int U = P / (int)gridDim.x;"),
]
SMS = (6, 7, 114, 132)
OLD_SUITE = ["tests/test_emu_kernels.py", "tests/test_emu_fuzz.py", "tests/test_emu_many_classes.py",
             "tests/test_emu_projection.py", "tests/test_emu_projection_conv1.py", "-k",
             "tensor or bank or fused or graphed or projection or conv1_matches or many"]
NEW_SUITE = ["tests/test_emu_sm_counts.py"]


def build_mutant(i, fname, old, new):
    out = f"/tmp/pcl_emu_sms_mutant_{i}"
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
    libs = {}
    procs = []
    for sms in SMS:
        libs[sms] = os.path.join(out, f"libpcl_emu_sm{sms}.so")
        procs.append(subprocess.Popen(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-ffp-contract=off",
                                       "-fno-strict-aliasing", "-w", "-Wno-psabi", f"-DPCL_EMU_SMS={sms}", "-I",
                                       os.path.join(b.HERE, "shim"), "-I", b.CSRC, "-I", os.path.join(b.ROOT, "include"),
                                       "-x", "c++"] + cpps + ["-o", libs[sms]]))
    assert all(p.wait() == 0 for p in procs), f"mutant {i}: build failed"
    return libs


def run_suite(libs, args):
    code = (f"import sys\nsys.path.insert(0, {os.path.join(ROOT, 'tests', 'emu')!r})\nimport build_emu\n"
            f"libs = {libs!r}\nbuild_emu.build = lambda force=False, sms=6: libs[sms]\nimport pytest\n"
            f"sys.exit(pytest.main({args + ['-q', '-x', '-p', 'no:cacheprovider']!r}))\n")
    return subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=3600).returncode


def check(i):
    name, fname, old, new = MUTANTS[i]
    libs = build_mutant(i, fname, old, new)
    rc_old, rc_new = run_suite(libs, OLD_SUITE), run_suite(libs, NEW_SUITE)
    how = lambda rc: "abort" if rc < 0 else ("killed" if rc else "survived")     # noqa: E731
    return name, how(rc_old), how(rc_new)


if __name__ == "__main__":
    with ThreadPoolExecutor(len(MUTANTS)) as ex:
        res = list(ex.map(check, range(len(MUTANTS))))
    for name, old, new in res:
        print(f"6-SM suite: {old:8s}  new tests: {new:8s}  {name}", flush=True)
    sys.exit(1 if any(new == "survived" for _, _, new in res) else 0)
