"""Mutation check of the captured criterion (tests/emu_fuzz.py: fuzz_graphed_criterion).

Each mutant changes ONE piece of what a GraphedContrastCriterion replay runs: the seg kernels of csrc/pcl_segce.cu
(built for the emulator, in a scratch copy of the sources) or the host code of graph_criterion.py / loss.py (a patched
copy of the package put first on sys.path).  Two suites run against every mutant:

  old  the emulated tests that reached this code before the criterion fuzzer: the seg-loss emulated tests
       (test_emu_ohem.py, test_emu_lovasz.py, test_emu_rmi.py), and test_emu_graphed_criterion.py and test_emu_fuzz.py
       with the fuzzer as of commit OLD_REV (read from git)
  new  the criterion fuzzer and its regression case in test_emu_fuzz.py

A suite kills a mutant when a test fails or the process aborts.  Nothing in the tree is modified.

One mutant is EQUIVALENT and runs as a control, expected to survive: pcl_seg_ce_fwd_bwd taking the two kernels at every
class count (segce_one_pass -> false).  That switch is a speed choice: the two forms give the same loss bits and a dseg
within 1e-6 max|g| of each other.  Its non-equivalent neighbour (the two-kernel branch dropping grad_scale) is in the
list.  The emulator runs the launch sequence eagerly, one kernel at a time: the graph's stream ordering and the real
atomics of the seg CE backward need the device fuzzer
(tests/test_gpu_graphed_criterion.py::test_fuzz_captured_criteria_on_the_device).

    python tools/emu_mutation_criterion.py      # one line per mutant; exit 1 if a mutant survives the new suite
"""
import os
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import build_emu as b  # noqa: E402

OLD_REV = "34fa8f0"          # the last commit without the criterion fuzzer
SEG, GC, LOSS = "pcl_segce.cu", "graph_criterion.py", "loss.py"
MUTANTS = [   # (name, file, exact text, replacement, equivalent)
    ("_Term: one_call when either dimension of the label grid is large enough", GC,
     "self.one_call = H >= h and W >= w", "self.one_call = H >= h or W >= w", False),
    ("_seg_half: the fp32 copy of a half head made for bf16 only (fp16 heads read stale logits)", GC,
     "            if x.dtype != torch.float32:\n                self.x32[k].copy_(x)",
     "            if x.dtype == torch.bfloat16:\n                self.x32[k].copy_(x)", False),
    ("set_grad_scale: the terms' coefficients ignored after a change", GC,
     "            t.set_grad_scale(value)", "            t.gs.fill_(float(value))", False),
    ("_total: the terms' coefficients left out of the total loss", GC,
     "v = t.loss if t.coef is None else t.coef * t.loss", "v = t.loss", False),
    ("seg_terms: the aux CE of the RMI / OHEM aux wrappers weighted with seg_loss", LOSS,
     'return [SegTerm("ce", "seg_aux", crit.ce_loss.ce_loss, lw["aux_loss"]), head]',
     'return [SegTerm("ce", "seg_aux", crit.ce_loss.ce_loss, lw["seg_loss"]), head]', False),
    ("pcl_seg_ce_fwd_bwd: the two kernels at every class count (speed choice)", SEG,
     "static bool segce_one_pass(int K) { return K <= KC_BWD_MAX; }",
     "static bool segce_one_pass(int K) { return false; }", True),
    ("pcl_seg_ce_fwd_bwd: the two-kernel branch (K > 24) without grad_scale", SEG,
     "return up_bwd_launch<k_segce_bwd_tile<false>>(a, s, dseg, (const float*)lse, (const float*)fin, grad_scale,",
     "return up_bwd_launch<k_segce_bwd_tile<false>>(a, s, dseg, (const float*)lse, (const float*)fin, nullptr,", False),
    ("k_segce_bwd_gather: every pixel ignored divides by the zero weight sum", SEG,
     "fin[1] == 0.f ? 0.f : acc * scale;", "acc * scale;", False),
    ("k_segce_scale: no early return for a zero weight sum", SEG,
     "  if (aw == 0.f) return;\n  const float scale = (grad_out", "  const float scale = (grad_out", False),
    ("k_lov_finalize: absent classes counted as present", SEG,
     "if (gts[c] > 0) { tot += s_d[0]; ++npres; }", "if (gts[c] >= 0) { tot += s_d[0]; ++npres; }", False),
    ("OHEM: the histogram reset narrowed to two of its three levels", SEG,
     "cudaMemsetAsync(hist, 0, (size_t)3 * OHEM_BINS * sizeof(int), s)",
     "cudaMemsetAsync(hist, 0, (size_t)2 * OHEM_BINS * sizeof(int), s)", False),
]
NEW_SUITE = ["tests/test_emu_fuzz.py::test_fuzz_graphed_criterion",
             "tests/test_emu_fuzz.py::test_criterion_fuzz_regression_two_call_ce_every_pixel_ignored"]
OLD_TESTS = ["tests/test_emu_ohem.py", "tests/test_emu_lovasz.py", "tests/test_emu_rmi.py"]


def old_suite(tmp):
    """The parent's fuzzer and its emulated criterion tests in `tmp` (imported before the tree's)."""
    for name in ("emu_fuzz.py", "test_emu_fuzz.py", "test_emu_graphed_criterion.py"):
        text = subprocess.run(["git", "show", f"{OLD_REV}:tests/{name}"], cwd=ROOT, capture_output=True, text=True,
                              check=True).stdout
        with open(os.path.join(tmp, name), "w") as f:
            f.write(text)
    return [os.path.join(tmp, "test_emu_fuzz.py"), os.path.join(tmp, "test_emu_graphed_criterion.py")] + OLD_TESTS


def build_mutant(i, fname, old, new):
    """(emulator library, directory to put first on sys.path or None) of mutant i."""
    out = f"/tmp/pcl_emu_criterion_mutant_{i}"
    shutil.rmtree(out, ignore_errors=True)
    os.makedirs(out)
    if fname.endswith(".py"):
        pkg = os.path.join(out, "contrastiveseg_b200")
        shutil.copytree(os.path.join(ROOT, "contrastiveseg_b200"), pkg,
                        ignore=shutil.ignore_patterns("__pycache__", "csrc"))
        path = os.path.join(pkg, fname)
        text = open(path).read()
        assert text.count(old) == 1, f"mutant {i}: source text not found once: {old}"
        with open(path, "w") as f:
            f.write(text.replace(old, new))
        return b.build(), out
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
    return lib, None


def run_suite(lib, args, pkg=None, first=None):
    pre = f"sys.path.insert(0, {pkg!r})\n" if pkg else ""
    if first:
        pre += f"sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})\nsys.path.insert(0, {first!r})\nimport emu_fuzz\n"
    code = (f"import sys\nsys.path.insert(0, {os.path.join(ROOT, 'tests', 'emu')!r})\nimport build_emu\n"
            f"build_emu.build = lambda force=False, sms=6: {lib!r}\n{pre}import contrastiveseg_b200\n"
            f"assert contrastiveseg_b200.__file__.startswith({(pkg or ROOT)!r}), contrastiveseg_b200.__file__\n"
            f"import pytest\n"
            f"sys.exit(pytest.main({args + ['-q', '-x', '-p', 'no:cacheprovider', '-m', 'not gpu']!r}))\n")
    return subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True,
                          timeout=7200).returncode


def check(i, tmp, old_args):
    name, fname, old, new, equivalent = MUTANTS[i]
    lib, pkg = build_mutant(i, fname, old, new)
    rc_old, rc_new = run_suite(lib, old_args, pkg, first=tmp), run_suite(lib, NEW_SUITE, pkg)
    how = lambda rc: "abort" if rc < 0 else ("killed" if rc else "survived")     # noqa: E731
    return name, how(rc_old), how(rc_new), equivalent


if __name__ == "__main__":
    b.build()
    with tempfile.TemporaryDirectory() as tmp:
        old_args = old_suite(tmp)
        with ThreadPoolExecutor(min(len(MUTANTS), max(1, (os.cpu_count() or 2) // 2))) as ex:
            res = list(ex.map(lambda i: check(i, tmp, old_args), range(len(MUTANTS))))
    for name, old, new, eq in res:
        print(f"old suite: {old:8s}  new suite: {new:8s}  {name}{'  (equivalent: control)' if eq else ''}", flush=True)
    sys.exit(1 if any(new == "survived" and not eq for _, _, new, eq in res) else 0)
