"""Mutation check of the embedding-width tests (tests/test_emu_widths.py) on the CPU emulator.

Each mutant changes ONE source text of the width-dependent arithmetic in a scratch copy of a kernel file or header.  Most
are faults that only show at widths the rest of the suite never runs: a bound or a count rounded to a power of two
(D & -D), a stride that is wrong for odd multiples of 32 (D & 32), a group count rounded down for a width that is not a
multiple of 8.  Each mutant is built for the emulator with tests/emu/build_emu.py (a mutated header goes into the mutant's
build directory, first on the include path) and run against two suites: the emulated tests that existed before
(test_emu_kernels.py, test_emu_fuzz.py, test_emu_mixed_precision.py, test_emu_many_classes.py) and
tests/test_emu_widths.py.  A suite kills a mutant when a test fails or the process aborts.  Mutants marked equivalent
compute the same values as the product by construction (the reason is printed); they are expected to survive both.
Nothing in the tree is modified.  Emulator only: a mutant is a deliberately wrong kernel and is never run on a GPU.

    python tools/emu_mutation_widths.py     # one line per mutant; exit 1 if a non-equivalent mutant survives the new tests
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import build_emu as b  # noqa: E402

SIMT, TILE, SEL, BANK = "pcl_infonce_simt.cu", "pcl_simt_tile.cuh", "pcl_select.cu", "pcl_bank.cu"
MUTANTS = [   # (name, source file, exact text, replacement, None or the reason the mutant is equivalent)
    ("load_tile_T: bound rounded down to a power of two", TILE,
     "for (int kk = kq * 8; kk < D; kk += 32)", "for (int kk = kq * 8; kk < (D & -D); kk += 32)", None),
    ("load_tile_T: stride 64 at odd multiples of 32", TILE,
     "for (int kk = kq * 8; kk < D; kk += 32)", "for (int kk = kq * 8; kk < D; kk += 32 + (D & 32))", None),
    ("k_sweep BWD: nq from D rounded down to a power of two", SIMT,
     "const int nq = D / 16;", "const int nq = (D & -D) / 16;", None),
    ("k_sweep BWD: accumulate guard q < nq widened to QMAX", SIMT,
     "          if (q < nq) {", "          if (q < QMAX) {",
     "the extra columns accumulate into dacc[i][q >= nq], which the guarded write never stores"),
    ("k_sweep BWD: write guard q < nq widened to QMAX", SIMT,
     "if (q < nq) dst[tx + 16 * q] = dacc[i][q];", "if (q < QMAX) dst[tx + 16 * q] = dacc[i][q];", None),
    ("simt_sweep_smem: D term rounded down to a power of two", SIMT,
     "return (size_t)(2 * D * LDT", "return (size_t)(2 * (D & -D) * LDT", None),
    ("k_scatter_reduce: 64 threads per row for D <= 128", SEL,
     "g->D <= 128 ? 128 : 256", "g->D <= 128 ? 64 : 256",
     "the channel loop strides by blockDim.x, and only the tensor path (D = 256) launches k_scatter_reduce"),
    ("k_zero_scatter: grid of B * (D rounded down to a power of two) planes", SEL,
     "const unsigned planes = (unsigned)(g->B * g->D);", "const unsigned planes = (unsigned)(g->B * (g->D & -g->D));",
     None),
    ("k_bank_segsum: channel groups D / 8 rounded down", BANK,
     "dim3(chunks, ceil_div(g->D, SEG_DG), g->B)", "dim3(chunks, g->D / SEG_DG, g->B)", None),
    ("k_bank_segsum: no early exit past the last channel", BANK,
     "    if (d0 + dl >= D) break;\n", "",
     "the flush writes only channels d0 + dl < D, so what the extra channels summed is dropped"),
    ("k_bank_rows: pixel row copy stops at the last full 32 lanes", BANK,
     "for (int dd = lane; dd < D; dd += 32) o[dd]", "for (int dd = lane; dd < (D & ~31); dd += 32) o[dd]", None),
]
OLD_SUITE = ["tests/test_emu_kernels.py", "tests/test_emu_fuzz.py", "tests/test_emu_mixed_precision.py",
             "tests/test_emu_many_classes.py"]
NEW_SUITE = ["tests/test_emu_widths.py"]


def mutate(i, text, old, new):
    assert text.count(old) == 1, f"mutant {i}: source text not found once: {old}"
    return text.replace(old, new)


def build_mutant(i):
    name, src, old, new, _ = MUTANTS[i]
    out = f"/tmp/pcl_emu_width_mutant_{i}"
    os.makedirs(out, exist_ok=True)
    for f in os.listdir(out):          # a header mutated by an earlier run must not shadow csrc/
        if f.endswith(".cuh"):
            os.remove(os.path.join(out, f))
    if src.endswith(".cuh"):           # out comes first on the include path
        with open(os.path.join(out, src), "w") as f:
            f.write(mutate(i, open(os.path.join(b.CSRC, src)).read(), old, new))
    cpps = []
    for fname in b.SOURCES:
        text = open(os.path.join(b.CSRC, fname)).read()
        if fname == src:
            text = mutate(i, text, old, new)
        p = os.path.join(out, fname[:-3] + ".emu.cpp")
        with open(p, "w") as f:
            f.write(b.rewrite(text))
        cpps.append(p)
    cpps.append(os.path.join(b.HERE, "emu_tc_stubs.cpp"))
    lib = os.path.join(out, "libpcl_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-ffp-contract=off", "-fno-strict-aliasing", "-w",
                    "-Wno-psabi", "-I", out, "-I", os.path.join(b.HERE, "shim"), "-I", b.CSRC, "-I",
                    os.path.join(b.ROOT, "include"), "-x", "c++"] + cpps + ["-o", lib], check=True)
    return lib


def run_suite(lib, files):
    """pytest over the files against the mutant library, four workers, stopping at the first failure; returns the exit
    code.  The library is swapped in by a plugin module that every worker process loads (-p)."""
    out = os.path.dirname(lib)
    with open(os.path.join(out, "emu_mutant_lib.py"), "w") as f:
        f.write(f"import sys\nsys.path.insert(0, {os.path.join(ROOT, 'tests', 'emu')!r})\nimport build_emu\n"
                f"build_emu.build = lambda force=False, sms=6: {lib!r}\n")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([out] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable, "-m", "pytest"] + files + ["-q", "-x", "-n", "4", "-p", "emu_mutant_lib", "-p", "no:cacheprovider"]
    return subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3600).returncode


if __name__ == "__main__":
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        libs = list(ex.map(build_mutant, range(len(MUTANTS))))
    how = lambda rc: "abort" if rc < 0 else ("killed" if rc else "survived")     # noqa: E731
    missed = 0
    for (name, _, _, _, equivalent), lib in zip(MUTANTS, libs):
        with ThreadPoolExecutor(2) as ex:
            rc_old, rc_new = ex.map(lambda files: run_suite(lib, files), (OLD_SUITE, NEW_SUITE))
        missed += rc_new == 0 and equivalent is None
        note = f"  (equivalent: {equivalent})" if equivalent else ""
        print(f"existing suite: {how(rc_old):8s}  new tests: {how(rc_new):8s}  {name}{note}", flush=True)
    sys.exit(1 if missed else 0)
