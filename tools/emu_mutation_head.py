"""Mutation check of the projection-head fuzzer (tests/emu_fuzz.py: fuzz_projection_head).

Each mutant changes ONE line of what the fused head runs: the column backward and conv1's epilogue in csrc/pcl_norm.cu
(built for the emulator, in a scratch copy of the sources) or the column hand-off in functional.py (a patched copy of
the package put first on sys.path).  No mutant indexes outside a tensor.  Two suites run against every mutant:

  old  the emulated tests that reached this code before the head fuzzer: test_emu_projection*.py,
       test_emu_sparse_head.py, and test_emu_fuzz.py with the fuzzer as of commit OLD_REV (read from git)
  new  the head fuzzer, its negative control, its regression and constructed edge cases in test_emu_fuzz.py

A suite kills a mutant when a test fails or the process aborts.  Nothing in the tree is modified.

One mutant is EQUIVALENT and runs as a control, expected to survive: is_placeholder without `len(self.deposits) == 1`.
deposit() appends to `deposits` and `zeros` together, so the remaining `len(self.zeros) == 1` decides the same.

    python tools/emu_mutation_head.py    # one line per mutant; exit 1 if a non-equivalent mutant survives the new suite
"""
import os
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emu_mutation_criterion as M  # noqa: E402

M.OLD_REV = "65627af"           # the last commit without the head fuzzer
NORM, FN = "pcl_norm.cu", "functional.py"
MUTANTS = [   # (name, file, exact text, replacement, equivalent)
    ("k_col_prep: the constant-1 column of gb2 not written", NORM,
     "  if (t == 0) ur[Cin] = 1.f;\n", "", False),
    ("k_col_prep: clamped anchors projected like the others (coef = dot)", NORM,
     "const float coef = inv < NORM_EPS_INV ? dot : 0.f;                                   // clamped rows",
     "const float coef = dot;                                   // clamped rows", False),
    ("k_col_prep: the channel loop over the first 256 channels only", NORM,
     "  for (int c = t; c < Cin; c += DOUT) {\n    const float yv",
     "  for (int c = t; c < Cin && c < DOUT; c += DOUT) {\n    const float yv", False),
    ("k_col_gemm<1>: the ReLU mask u > 0 taken as u >= 0", NORM,
     "o.u[(int64_t)i * (o.Cin + 1) + j] > 0.f ? acc[r][c] : 0.f;",
     "o.u[(int64_t)i * (o.Cin + 1) + j] >= 0.f ? acc[r][c] : 0.f;", False),
    ("k_bn_input_grad_cols: the k1 term dropped", NORM,
     "gr[p] = from_f32<T>(k.a * (0.f - k.k1 - (yv[i] - k.mu) * k.k2));",
     "gr[p] = from_f32<T>(k.a * (0.f - (yv[i] - k.mu) * k.k2));", False),
    ("k_bn_cols_scatter: g_u written without the BN terms", NORM,
     "g[o] = from_f32<T>(k.a * (gu - k.k1 - (to_f32(y[o]) - k.mu) * k.k2));", "g[o] = from_f32<T>(k.a * gu);", False),
    ("k_conv1_gemm: tail-tile pixels beyond HW summed into the BN statistics (store still guarded)", NORM,
     "        if (p0 + px < a.HW) {\n          const T v = stage[cl * LD + px];\n"
     "          out[(int64_t)c * a.HW + p0 + px] = v;",
     "        {\n          const T v = stage[cl * LD + px];\n"
     "          if (p0 + px < a.HW) out[(int64_t)c * a.HW + p0 + px] = v;", False),
    ("_with_deposits: the deposits added without rounding to zn's dtype", FN,
     "gv[b, :, p] += cols[live].to(dtype)", "gv[b, :, p] += cols[live]", False),
    ("is_placeholder: without len(self.deposits) == 1 (deposit() appends to both lists)", FN,
     "return (len(self.deposits) == 1 and len(self.zeros) == 1", "return (len(self.zeros) == 1", True),
    ("is_placeholder: every stride 0 again (a W = 1 map silently takes the dense path)", FN,
     "all(st == 0 or n == 1 for st, n in zip(g.stride(), g.shape))", "all(st == 0 for st in g.stride())", False),
]
NEW_SUITE = ["tests/test_emu_fuzz.py::test_fuzz_projection_head",
             "tests/test_emu_fuzz.py::test_head_fuzz_detects_a_weight_packed_once",
             "tests/test_emu_fuzz.py::test_head_fuzz_regression_column_path_at_width_one",
             "tests/test_emu_fuzz.py::test_head_fuzz_edge_cases"]
OLD_TESTS = ["tests/test_emu_projection.py", "tests/test_emu_projection_bf16.py", "tests/test_emu_projection_bnrelu.py",
             "tests/test_emu_projection_conv1.py", "tests/test_emu_sparse_head.py"]


def old_suite(tmp):
    """The parent's fuzzer and its emulated fuzz tests in `tmp` (imported before the tree's)."""
    import subprocess
    for name in ("emu_fuzz.py", "test_emu_fuzz.py"):
        text = subprocess.run(["git", "show", f"{M.OLD_REV}:tests/{name}"], cwd=ROOT, capture_output=True, text=True,
                              check=True).stdout
        with open(os.path.join(tmp, name), "w") as f:
            f.write(text)
    return [os.path.join(tmp, "test_emu_fuzz.py")] + OLD_TESTS


if __name__ == "__main__":
    M.MUTANTS, M.NEW_SUITE = MUTANTS, NEW_SUITE
    M.b.build()
    with tempfile.TemporaryDirectory() as tmp:
        old_args = old_suite(tmp)
        with ThreadPoolExecutor(min(len(MUTANTS), max(1, (os.cpu_count() or 2) // 2))) as ex:
            res = list(ex.map(lambda i: M.check(i, tmp, old_args), range(len(MUTANTS))))
    for name, old, new, eq in res:
        print(f"old suite: {old:8s}  new suite: {new:8s}  {name}{'  (equivalent: control)' if eq else ''}", flush=True)
    sys.exit(1 if any(new == "survived" and not eq for _, _, new, eq in res) else 0)
