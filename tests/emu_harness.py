"""TEST INFRASTRUCTURE: run the Python layer against the host-thread build of the SIMT kernels (tests/emu) on CPU
tensors.  `use_emulation(monkeypatch)` swaps the loaded library and the few CUDA-only hooks of the host layer."""
import ctypes as C
import os
import sys
import types

import torch

from contrastiveseg_b200 import _abi, bank as bank_mod, functional as Fn

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import build_emu  # noqa: E402

_libs = {}


def emu_library(sms: int = 6):
    """The emulator library for an `sms`-SM device, loaded once per count (each count is a library of its own)."""
    if sms not in _libs:
        lib = C.CDLL(build_emu.build() if sms == 6 else build_emu.build(sms=sms))
        for name, (res, args) in _abi.SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        assert lib.pcl_emulated() == 1
        _libs[sms] = lib
    return _libs[sms]


class _NoCtx:
    def __init__(self, *a, **k):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


def use_emulation(monkeypatch, sms: int = 6):
    lib = emu_library(sms)
    monkeypatch.setattr(_abi, "load", lambda *a, **k: lib)
    monkeypatch.setattr(Fn, "_require_cuda", lambda t, name: None)
    monkeypatch.setattr(Fn, "_stream_ptr", lambda device: 0)
    monkeypatch.setattr(Fn, "_on_device", _NoCtx)
    monkeypatch.setattr(bank_mod, "_is_cuda", lambda t: True)
    monkeypatch.setattr(torch.cuda, "device", _NoCtx)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: types.SimpleNamespace(cuda_stream=0))
    orig_init = Fn.ContrastWorkspace.__init__

    def init(self, *a, **k):
        orig_init(self, *a, **k)
        self.ranks_host = torch.zeros_like(self.ranks)          # pinned staging buffer on a CUDA box

    monkeypatch.setattr(Fn.ContrastWorkspace, "__init__", init)
    if os.environ.get("PCL_EMU_POISON"):
        # uninitialised-read check: every torch.empty / empty_like buffer (scratch AND outputs) starts as NaN / a large
        # integer instead of whatever the allocator returns; a kernel that reads scratch it never wrote poisons its result
        real_empty, real_empty_like = torch.empty, torch.empty_like

        def _poison(t):
            if t.numel():
                with torch.no_grad():
                    if t.dtype.is_floating_point:
                        t.fill_(float("nan"))
                    elif t.dtype in (torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64):
                        t.fill_(torch.iinfo(t.dtype).max - 7)
            return t

        monkeypatch.setattr(torch, "empty", lambda *a, **k: _poison(real_empty(*a, **k)))
        monkeypatch.setattr(torch, "empty_like", lambda *a, **k: _poison(real_empty_like(*a, **k)))
    Fn.clear_workspaces()
    Fn._BANK_READERS.clear()
    return lib
