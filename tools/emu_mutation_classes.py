"""Mutation check of the many-class tests (tests/test_emu_many_classes.py) on the CPU emulator.

Each mutant changes ONE source text in a scratch copy of a kernel file or header (a class-chunk offset dropped from the
seg-CE kernels or from the patch staging every up-sampling loss shares, the K > 32 argmax turned into a last-maximum, the
plan's shared-memory table bound raised past its size), is built for the emulator with tests/emu/build_emu.py and must
make the emulated many-class tests fail or abort.  A mutated header is written to the mutant's build directory, which
comes first on the include path.  Nothing in the tree is modified.  The last mutant (the plan keeps 9 x 512 totals in its 4096-entry shared table) is caught by
the emulator's index check of fixed-size __shared__ arrays (emu::SharedArray): the B = 9, K = 256 plan case aborts at
the first write past the table.  Emulator only: a mutant is a deliberately wrong kernel and is never run on a GPU.

    python tools/emu_mutation_classes.py              # one line per mutant and the new tests that kill it; exit 1 if any survives
    python tools/emu_mutation_classes.py --existing   # also report whether test_emu_kernels.py / test_emu_fuzz.py kill it
"""
import os
import re
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import build_emu as b  # noqa: E402

MUTANTS = [   # (name, source file, exact text, replacement, which occurrence)
    ("segce fwd: target compare without the chunk offset", "pcl_segce.cu",
     "if (c0 + cc == (int)t) vt = v;", "if (cc == (int)t) vt = v;", 0),
    ("segce bwd tile: one-hot without the chunk offset", "pcl_segce.cu",
     "((c0 + cc) == (int)t ? 1.f : 0.f)", "(cc == (int)t ? 1.f : 0.f)", 0),
    ("segce bwd tile: dseg flush without the chunk offset", "pcl_segce.cu",
     "dseg + ((int64_t)b * a.K + c0) * hw", "dseg + ((int64_t)b * a.K) * hw", 0),
    ("up_stage: staged load without the chunk offset", "pcl_upsample.cuh",
     "S[cc * pitch + r] = seg[((int64_t)b * a.K + c0 + cc) * hw", "S[cc * pitch + r] = seg[((int64_t)b * a.K + cc) * hw", 0),
    ("select k_keys K > 32: last maximum wins", "pcl_select.cu",
     "if (v[u] > best) { best = v[u]; pred = c0 + u; }", "if (v[u] >= best) { best = v[u]; pred = c0 + u; }", 0),
    ("select fused tail: shared totals past the 4096-entry table", "pcl_select.cu",
     "rows <= 4096", "rows <= 8192", 0),
]
NEW = os.path.join(ROOT, "tests", "test_emu_many_classes.py")
EXISTING = [os.path.join(ROOT, "tests", "test_emu_kernels.py"), os.path.join(ROOT, "tests", "test_emu_fuzz.py")]


def mutate(idx, text, needle, repl, occ):
    assert text.count(needle) > occ, f"mutant {idx}: occurrence {occ} of the source text not found: {needle}"
    at = -1
    for _ in range(occ + 1):
        at = text.index(needle, at + 1)
    return text[:at] + repl + text[at + len(needle):]


def build_mutant(idx, src, needle, repl, occ, out):
    os.makedirs(out, exist_ok=True)
    for f in os.listdir(out):          # a header mutated by an earlier run must not shadow csrc/
        if f.endswith(".cuh"):
            os.remove(os.path.join(out, f))
    if src.endswith(".cuh"):           # out comes first on the include path
        with open(os.path.join(out, src), "w") as f:
            f.write(mutate(idx, open(os.path.join(b.CSRC, src)).read(), needle, repl, occ))
    cpps = []
    for name in b.SOURCES:
        text = open(os.path.join(b.CSRC, name)).read()
        if name == src:
            text = mutate(idx, text, needle, repl, occ)
        p = os.path.join(out, name[:-3] + ".emu.cpp")
        with open(p, "w") as f:
            f.write(b.rewrite(text))
        cpps.append(p)
    cpps.append(os.path.join(b.HERE, "emu_tc_stubs.cpp"))
    lib = os.path.join(out, "libpcl_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-ffp-contract=off", "-fno-strict-aliasing", "-w", "-Wno-psabi",
                    "-I", out, "-I", os.path.join(b.HERE, "shim"), "-I", b.CSRC, "-I", os.path.join(b.ROOT, "include"), "-x", "c++"] + cpps +
                   ["-o", lib], check=True)
    return lib


def run_tests(lib, files):
    """Run the test files against the mutant library; returns (exit code, ids of the failed tests)."""
    code = (f"import sys\nsys.path.insert(0, {os.path.join(ROOT, 'tests', 'emu')!r})\nimport build_emu\n"
            f"build_emu.build = lambda force=False: {lib!r}\nimport pytest\n"
            f"sys.exit(pytest.main({files!r} + ['-q', '-rf', '-p', 'no:cacheprovider']))\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=3600)
    failed = re.findall(r"^FAILED \S+::(\S+)", r.stdout, re.M)
    return r.returncode, failed


if __name__ == "__main__":
    existing = "--existing" in sys.argv[1:]
    survivors = 0
    for i, (name, src, needle, repl, occ) in enumerate(MUTANTS):
        lib = build_mutant(i, src, needle, repl, occ, f"/tmp/pcl_emu_class_mutant_{i}")
        rc, failed = run_tests(lib, [NEW])
        killed = rc != 0
        survivors += 0 if killed else 1
        how = "abort" if rc < 0 else ("fail" if rc else "pass")
        line = f"{'killed  ' if killed else 'SURVIVED'} [{how}]  {name}: {', '.join(failed) or '-'}"
        if existing:
            rc_old, failed_old = run_tests(lib, EXISTING)
            line += f"  | existing emulated suite: {'killed' if rc_old else 'survived'} ({len(failed_old)} failed)"
        print(line, flush=True)
    sys.exit(1 if survivors else 0)
