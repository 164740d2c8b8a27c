"""Mutation check of the CPU emulator's power to catch pipeline-protocol bugs in the tensor path (tests/emu).

Each mutant removes ONE mbarrier wait from a scratch copy of csrc/pcl_infonce_tc.cu (a consumer no longer waits for its
data, a producer no longer waits for a free stage, ...), is built for the emulator and must make the emulated tensor tests
fail or abort.  A mutant that survives marks a blind spot of the model.  Nothing in the tree is modified.  The ring wait
and the producer are shared by k_tc_fwd and k_tc_pos_t, so those mutants break both kernels.

    python tools/emu_mutation.py            # prints one line per mutant, exit 1 if any survives
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
import build_emu as b  # noqa: E402

MUTANTS = [   # (name, exact source text to delete: found once in csrc/pcl_infonce_tc.cu)
    ("ring_mma: no wait for the ring stage (full)", "ptx::mbar_wait(&full[ring.stage], ring.phase);"),
    ("producer: no wait for a free ring stage (empty)", "ptx::mbar_wait(&sm.empty[p.stage], p.phase ^ 1);"),
    ("producer: no wait for the previous item's MMAs (a_empty)", "ptx::mbar_wait(&sm.a_empty, (p.item - 1) & 1);"),
    ("k_tc_fwd consumers: no wait for the anchor tile (a_full)", "ptx::mbar_wait(&sm.a_full, seg_idx & 1);"),
    ("k_tc_pos_t consumers: no wait for the anchor block (a_full)", "ptx::mbar_wait(&sm.a_full, seq & 1);"),
    ("k_tc_bwd producer: no wait for a free contrast stage (c_empty)", "ptx::mbar_wait(&sm.c_empty[stage], phase ^ 1);"),
    ("k_tc_bwd consumers: no wait for the contrast tile (c_full)", "ptx::mbar_wait(&sm.c_full[stage], phase);"),
    ("k_tc_bwd consumers: no wait for the anchor tile (a_full)", "ptx::mbar_wait(&sm.a_full, 0);"),
]
TESTS = ("tc_pipeline_raw_logits or tc_forward_matches_oracle or tc_backward_matches_oracle or loss_module_on_tensor_path "
         "or by_class_blocks or graphed_bank")


def build_mutant(idx, needle, out):
    os.makedirs(out, exist_ok=True)
    cpps = []
    for name in b.SOURCES:
        text = open(os.path.join(b.CSRC, name)).read()
        if name == "pcl_infonce_tc.cu":
            assert text.count(needle) == 1, f"mutant {idx}: source text not found once: {needle}"
            text = text.replace(needle, "/* mutant: wait removed */")
        p = os.path.join(out, name[:-3] + ".emu.cpp")
        with open(p, "w") as f:
            f.write(b.rewrite(text))
        cpps.append(p)
    cpps.append(os.path.join(b.HERE, "emu_tc_stubs.cpp"))
    lib = os.path.join(out, "libpcl_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-ffp-contract=off", "-fno-strict-aliasing", "-w", "-Wno-psabi", "-I",
                    os.path.join(b.HERE, "shim"), "-I", b.CSRC, "-I", os.path.join(b.ROOT, "include"), "-x", "c++"] + cpps +
                   ["-o", lib], check=True)
    return lib


def run_tests(lib, delay, sched=None):
    code = (f"import sys\nsys.path.insert(0, {os.path.join(ROOT, 'tests', 'emu')!r})\nimport build_emu\n"
            f"build_emu.build = lambda force=False: {lib!r}\nimport pytest\n"
            f"sys.exit(pytest.main([{os.path.join(ROOT, 'tests', 'test_emu_kernels.py')!r}, '-q', '-x', '-p', 'no:cacheprovider', "
            f"'-k', {TESTS!r}]))\n")
    env = dict(os.environ, PCL_EMU_ASYNC_DELAY=str(delay))
    if sched:
        env["PCL_EMU_SCHED"] = sched          # random thread order + out-of-order / partial TMA completion
    return subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900).returncode


def check(i):
    name, needle = MUTANTS[i]
    lib = build_mutant(i, needle, f"/tmp/pcl_emu_mutant_{i}")
    rcs = [run_tests(lib, 1), run_tests(lib, 4), run_tests(lib, 1, "random:5"), run_tests(lib, 2, "random:77")]
    return name, rcs


if __name__ == "__main__":
    with ThreadPoolExecutor(len(MUTANTS)) as ex:
        res = list(ex.map(check, range(len(MUTANTS))))
    survivors = 0
    for name, rcs in res:
        killed = any(rc != 0 for rc in rcs)
        survivors += 0 if killed else 1
        how = "/".join("abort" if rc < 0 else ("fail" if rc else "pass") for rc in rcs)
        print(f"{'killed  ' if killed else 'SURVIVED'} [{how}]  {name}", flush=True)
    sys.exit(1 if survivors else 0)
