"""interaction._launch, the one path from the wrappers into the library, against a fake library entry (no GPU): the
arguments it passes, that it keeps temporaries alive through the call, and that a failed call raises naming the entry."""
import contextlib
import ctypes
import types
import weakref

import pytest
import torch

from matchmaker_b200 import _lib, interaction

STREAM = 0x5EED
DEV = torch.device("cuda", 0)


@pytest.fixture
def fake_lib(monkeypatch):
    """_lib.load() returns a namespace; the device context and the current stream need no device."""
    lib = types.SimpleNamespace(mmb200_last_error=lambda: b"fake failure")
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda dev: types.SimpleNamespace(cuda_stream=STREAM))
    return lib


def _entry(lib, argtypes, body):
    body.argtypes = argtypes
    lib.mmb200_fake = body


def test_tensors_become_pointers_and_none_null(fake_lib):
    calls = []
    _entry(fake_lib, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p],
           lambda *a: calls.append(a) or 0)
    t, n = torch.arange(6.0), torch.tensor(7)
    interaction._launch(DEV, "mmb200_fake", t, None, 3, n, 0.5)
    # a tensor in a scalar slot is passed as given (ctypes takes a 0-dim integer tensor as its value)
    assert calls == [(t.data_ptr(), None, 3, n, 0.5, STREAM)]


def test_a_temporary_argument_lives_until_the_call_returns(fake_lib):
    refs, alive = [], []
    _entry(fake_lib, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p],
           lambda *a: alive.append([r() is not None for r in refs]) or 0)

    def temporary(t):
        c = t.contiguous()
        refs.append(weakref.ref(c))
        return c

    base = torch.arange(12.0).view(3, 4)
    interaction._launch(DEV, "mmb200_fake", temporary(base.t()), temporary(base[:, ::2]))
    assert alive == [[True, True]]
    assert all(r() is None for r in refs)   # released once the call has returned


def test_a_failed_call_raises_naming_the_entry(fake_lib):
    _entry(fake_lib, [ctypes.c_int64, ctypes.c_void_p], lambda *a: _lib.ERR_INVALID)
    with pytest.raises(_lib.MatchmakerB200Error, match=r"^mmb200_fake: invalid argument \(-1\): fake failure$"):
        interaction._launch(DEV, "mmb200_fake", 1)
