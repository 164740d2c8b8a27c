"""TEST INFRASTRUCTURE: build tests/emu/_build/libpcl_emu.so — the engine's SIMT kernel sources compiled for host
threads (fibers) with g++, so CPU-only test runs execute the real kernel code.  See shim/cuda_runtime.h.

Source rewriting (text level, the .cu files themselves are untouched):
  kernel<<<grid, block, smem, stream>>>(args)   ->  emu::cfg(grid, block, smem, stream).bind(kernel)(args)
  extern __shared__ [__align__(n)] T name[];     ->  T* name = reinterpret_cast<T*>(emu::dyn_smem());
  __shared__ T a[N], b[M];                       ->  __shared__ emu::SharedArray<T, (N)> a; ... (index checked)
  asm volatile("bar.sync id, %0;" :: "n"(N) ...) ->  emu::named_barrier(id, N);
The tensor path (pcl_infonce_tc.cu, pcl_infonce_fused.cu) compiles against shim/ptx_sm90.cuh, a functional model of the
mbarrier / TMA / wgmma primitives with the product header's names (found first on the include path).
"""
from __future__ import annotations

import hashlib
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
CSRC = os.path.join(ROOT, "contrastiveseg_b200", "csrc")
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(BUILD, "libpcl_emu.so")
SOURCES = ["pcl_api.cu", "pcl_select.cu", "pcl_infonce_simt.cu", "pcl_topk.cu", "pcl_graph.cu", "pcl_bank.cu",
           "pcl_norm.cu", "pcl_segce.cu", "pcl_step.cu", "pcl_infonce_tc.cu", "pcl_infonce_fused.cu"]

LAUNCH = re.compile(r"([A-Za-z_][\w:]*(?:<[^<>;()]*>)?)\s*<<<(.*?)>>>", re.S)
NAMED_BARRIER = re.compile(r'asm volatile\("bar\.sync (\d+), %0;" ::"n"\((\w+)\) : "memory"\);')
EXTERN_SHARED = re.compile(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?([A-Za-z_][\w ]*?)\s+(\w+)\s*\[\s*\]\s*;")
# fixed-size 1-D __shared__ arrays, one or several declarators: `__shared__ float a[N], b[M];`
FIXED_SHARED = re.compile(r"__shared__\s+([A-Za-z_][\w ]*?)\s+((?:\w+\s*\[[^\[\];]+\]\s*,\s*)*\w+\s*\[[^\[\];]+\])\s*;")
DECLARATOR = re.compile(r"(\w+)\s*\[([^\[\];]+)\]")


def _checked_shared(m: re.Match) -> str:
    return " ".join(f"__shared__ emu::SharedArray<{m.group(1)}, ({n})> {name};" for name, n in DECLARATOR.findall(m.group(2)))


def rewrite(text: str) -> str:
    text = EXTERN_SHARED.sub(lambda m: f"{m.group(1)}* {m.group(2)} = reinterpret_cast<{m.group(1)}*>(emu::dyn_smem());", text)
    text = FIXED_SHARED.sub(_checked_shared, text)
    text = NAMED_BARRIER.sub(lambda m: f"emu::named_barrier({m.group(1)}, {m.group(2)});", text)
    return LAUNCH.sub(lambda m: f"emu::cfg({m.group(2)}).bind({m.group(1)})", text)


def _digest() -> str:
    h = hashlib.sha256()
    for d in (CSRC, os.path.join(ROOT, "include"), HERE, os.path.join(HERE, "shim")):
        for f in sorted(os.listdir(d)):
            if f.endswith((".cu", ".cuh", ".h", ".cpp", ".py")):
                h.update(f.encode())
                h.update(open(os.path.join(d, f), "rb").read())
    return h.hexdigest()


def build(force: bool = False, sms: int = 6) -> str:
    """The emulator library modelling an `sms`-SM device.  6 SMs (the suite's default) is libpcl_emu.so; other counts get
    a library of their own (libpcl_emu_sm<n>.so), because pcl::num_sms() caches the count per process."""
    lib = LIB if sms == 6 else os.path.join(BUILD, f"libpcl_emu_sm{sms}.so")
    stamp = os.path.join(BUILD, "build.sha256" if sms == 6 else f"build_sm{sms}.sha256")
    dig = _digest()
    if not force and os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read() == dig:
        return lib
    os.makedirs(BUILD, exist_ok=True)
    cpps = []
    for name in SOURCES:
        out = os.path.join(BUILD, name[:-3] + ".emu.cpp")
        text = f'#line 1 "{os.path.join(CSRC, name)}"\n' + rewrite(open(os.path.join(CSRC, name)).read())
        if not (os.path.exists(out) and open(out).read() == text):     # (builds of several counts share these files)
            with open(out, "w") as f:
                f.write(text)
        cpps.append(out)
    cpps.append(os.path.join(HERE, "emu_tc_stubs.cpp"))
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-ffp-contract=off", "-fno-strict-aliasing", "-w",
           f"-DPCL_EMU_SMS={int(sms)}", "-I", os.path.join(HERE, "shim"), "-I", CSRC, "-I", os.path.join(ROOT, "include"),
           "-x", "c++"] + cpps + ["-o", lib]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("emulation build failed:\n" + r.stdout[-4000:] + r.stderr[-8000:])
    with open(stamp, "w") as f:
        f.write(dig)
    return lib


if __name__ == "__main__":
    print(build(force=True))
