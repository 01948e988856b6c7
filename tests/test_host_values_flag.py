"""KB_CFG_HOST_VALUES without a GPU: the header defines it, and Engine(host_values=True) hands it to kb_open."""
from __future__ import annotations

import ctypes as C
import os
import re

import pytest

from kubebrain_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_define(name: str) -> int:
    src = open(os.path.join(ROOT, "include", "kb_b200.h")).read()
    m = re.search(r"#define\s+%s\s+(\d+)u?\b" % name, src)
    assert m, name
    return int(m.group(1))


def test_header_defines_the_flags():
    assert _header_define("KB_CFG_HOST_VALUES") == _lib.KB_CFG_HOST_VALUES == 2
    assert _header_define("KB_CFG_HIGH_PRIORITY") == _lib.KB_CFG_HIGH_PRIORITY
    assert "int kb_store_mem(kb_ctx *ctx, uint64_t *device_bytes, uint64_t *host_bytes);" in open(
        os.path.join(ROOT, "include", "kb_b200.h")).read()


class _FakeLib:
    """stands in for libkbb200.so: records the kb_config kb_open receives and refuses to open"""

    def __init__(self):
        self.seen = []

    def kb_open(self, device, cfg, out):
        c = C.cast(cfg, C.POINTER(_lib.KbConfig)).contents
        self.seen.append((device, c.struct_size, c.flags))
        return _lib.KB_ECUDA

    def kb_close(self, ctx):
        pass


@pytest.mark.parametrize("high,host,flags", [(False, False, 0), (False, True, 2), (True, False, 1), (True, True, 3)])
def test_engine_passes_the_flags(monkeypatch, high, host, flags):
    fake = _FakeLib()
    monkeypatch.setattr(_lib, "lib", lambda: fake)
    with pytest.raises(_lib.KbError):
        _lib.Engine(1, high_priority=high, host_values=host)
    assert fake.seen == [(1, C.sizeof(_lib.KbConfig), flags)]
