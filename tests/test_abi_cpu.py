"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol
include/simdjson_b200.h declares, refuses to work without a device (no CPU fallback), and its
host-only helper agrees with the oracle.  No compute calls here."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from simdjson_b200 import _lib
    return _lib.load()


def _declared():
    src = open(os.path.join(ROOT, "include", "simdjson_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sj_[a-z0-9_]+)\s*\(", src)))


def test_every_declared_symbol_is_exported(lib):
    from simdjson_b200 import _lib
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), "missing export " + n
    assert sorted(_lib.EXPORTS) == names


def test_python_mirror_uses_the_headers_numbers(lib):
    """return codes, flags and the exchange handle size of the ctypes mirror are the header's #defines; sj_error_string knows
    every code"""
    from simdjson_b200 import _lib
    src = open(os.path.join(ROOT, "include", "simdjson_b200.h")).read()
    defs = {k: int(v.rstrip("u"), 0) for k, v in re.findall(r"#define\s+(SJ_[A-Z0-9_]+)\s+(0x[0-9a-fA-F]+u?|[0-9]+u?)\b", src)}
    for name, val in (("SJ_OK", _lib.OK), ("SJ_ERR_STAGE1", _lib.ERR_STAGE1), ("SJ_ERR_STAGE2", _lib.ERR_STAGE2),
                      ("SJ_ERR_NO_DEVICE", _lib.ERR_NO_DEVICE), ("SJ_ERR_CAPACITY", _lib.ERR_CAPACITY),
                      ("SJ_ERR_TOO_LARGE", _lib.ERR_TOO_LARGE), ("SJ_ERR_ARGUMENT", _lib.ERR_ARGUMENT),
                      ("SJ_ERR_EXCHANGE", _lib.ERR_EXCHANGE), ("SJ_ERR_PEER", _lib.ERR_PEER),
                      ("SJ_FLAG_NDJSON", _lib.FLAG_NDJSON), ("SJ_FLAG_COPY_STRINGS", _lib.FLAG_COPY_STRINGS),
                      ("SJ_EXCHANGE_HANDLE_BYTES", _lib.EXCHANGE_HANDLE_BYTES)):
        assert defs[name] == val, name
    lib.sj_error_string.restype = C.c_char_p
    codes = [v for k, v in defs.items() if k.startswith(("SJ_ERR_", "SJ_STREAM_")) or k == "SJ_OK"]
    assert len(set(codes)) == len(codes)  # no two codes share a number
    for v in codes:
        assert lib.sj_error_string(v) not in (None, b"", b"unknown error"), v


def test_exchange_needs_a_context(lib):
    """the exchange entry points take a context that owns an exchange: without one they refuse (no device here, so no
    context can exist) instead of touching memory"""
    assert lib.sj_exchange_create(None, 0, 2, 1, None) != 0
    assert lib.sj_exchange_connect(None, None) != 0
    assert lib.sj_exchange_connect_ptrs(None, None) != 0
    assert lib.sj_exchange_set_gap(None, 1) != 0
    assert lib.sj_exchange_set_timeout_ms(None, 1000) != 0
    assert not lib.sj_exchange_local(None) and not lib.sj_exchange_bases(None)
    out = (C.c_uint64 * 10)()
    assert lib.sj_exchange_result(None, out) != 0


def test_no_device_means_no_service(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    assert lib.sj_supported() == 0
    h = C.c_void_p()
    assert lib.sj_ctx_create(0, C.byref(h)) == 3  # SJ_ERR_NO_DEVICE: the product path has no CPU fallback
    assert not h.value


def test_trim_space_matches_oracle(lib, oracle):
    cases = [b"  {} \n", b"\xc2\xa0{}\xe2\x80\x83", b"\xff {} ", b" \t\r\n", b"\x0b\x0c[]\xe3\x80\x80", b"{}\xc2",
             b"\xe1\x9a\x80[1]\xc2\x85", b"", b"x", b"\xe2\x80\x8a[\xe2\x80\x8b]\xe2\x80\xa8"]
    for src in cases:
        a, b = C.c_size_t(0), C.c_size_t(0)
        buf = (C.c_uint8 * max(1, len(src))).from_buffer_copy(src or b"\0")
        lib.sj_trim_space(buf, len(src), C.byref(a), C.byref(b))
        assert (a.value, b.value) == oracle.trim_space(src), src


def test_header_is_plain_c_and_links_from_c(lib, tmp_path):
    """include/simdjson_b200.h compiled by a C11 compiler with -Werror, linked against the library from plain C
    (what cgo sees); without a device the example stops at SJ_ERR_NO_DEVICE -- no CPU fallback"""
    import subprocess
    import torch
    exe = str(tmp_path / "abi_example")
    libdir = os.path.join(ROOT, "simdjson-go_b200")
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tools", "abi_example.c"), "-L" + libdir, "-lsimdjson_b200",
                           "-Wl,-rpath," + libdir, "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert "trimmed window: [1, 49)" in out.stdout, out.stdout + out.stderr
    if not torch.cuda.is_available():
        assert out.returncode == 3 and "no sm_90 device" in out.stdout, out.stdout + out.stderr
