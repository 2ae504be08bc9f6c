"""The C-ABI shared library: loads, exports every symbol include/b200vit.h declares, rejects bad arguments with an
error code + message (no compute, no GPU needed)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT
from vit_pytorch_b200 import _lib, build


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        build.build()
    return _lib.lib()


def header_functions():
    src = open(os.path.join(ROOT, "include", "b200vit.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200vit_\w+)\s*\(", src)))


def test_header_symbols_are_exported(lib):
    names = header_functions()
    assert len(names) >= 12
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/b200vit.h but not exported"
    assert set(_lib.SYMBOLS) <= set(names)


def test_version_and_launch_counter(lib):
    assert lib.b200vit_version() >= 100
    assert lib.b200vit_stats_parts(768) == 6 and lib.b200vit_stats_parts(128) == 2 and lib.b200vit_stats_parts(1000) == 8
    lib.b200vit_reset_launch_count()
    assert lib.b200vit_launch_count() == 0


def test_bad_arguments_return_error_codes(lib):
    rc = lib.b200vit_gemm_bf16(None, 8, None, 8, None, None, 8, None, None, None, 0, 1e-5, None, None, 1, 1, 8, 0, None)
    assert rc == -1 and b"null" in lib.b200vit_last_error()
    rc = lib.b200vit_attention(ctypes.c_void_p(256), ctypes.c_void_p(256), 1, 16, 1, 96, 0.1, None)
    assert rc == -1 and b"dim_head=96" in lib.b200vit_last_error()
    rc = lib.b200vit_attention(ctypes.c_void_p(256), ctypes.c_void_p(256), 1, 4096, 1, 64, 0.1, None)
    assert rc == -1 and b"512" in lib.b200vit_last_error()     # single-pass kernel; longer: b200vit_attention_varlen
    rc = lib.b200vit_patchify_ln(ctypes.c_void_p(256), ctypes.c_void_p(256), ctypes.c_void_p(256), ctypes.c_void_p(256),
                                 64, 1, 3, 30, 32, 4, 4, 1e-5, None)
    assert rc == -1 and b"divisible" in lib.b200vit_last_error()
    # one-call encoder: argument checks happen before any device work
    layers = (_lib.Layer * 1)()
    ws = _lib.EncoderWs()
    rc = lib.b200vit_encoder_blocks(layers, 1, ctypes.c_void_p(256), ctypes.byref(ws), 1, 16, 64, 1, 64, 128, 0.125, 0,
                                    None, None, 0, None)
    assert rc == -1 and b"workspace" in lib.b200vit_last_error()
    full = _lib.EncoderWs(*([256] * 7))
    rc = lib.b200vit_encoder_blocks(layers, 1, ctypes.c_void_p(256), ctypes.byref(full), 1, 600, 64, 1, 64, 128, 0.125,
                                    1, None, None, 0, None)
    assert rc == -1 and b"varlen" in lib.b200vit_last_error()
    assert ctypes.sizeof(_lib.Layer) == 11 * 8 + 8 and ctypes.sizeof(_lib.EncoderWs) == 7 * 8   # as the C structs


def test_debug_set_accepts_only_the_documented_hooks(lib):
    """Keys 12, 14 and 15 are the test hooks include/b200vit.h lists (set to their defaults here); any other key is
    B200VIT_ERR_INVALID."""
    for key in (12, 14, 15):
        assert lib.b200vit_debug_set(key, 0) == 0, key
    for key in (1, 11, 13, 0, 16):
        assert lib.b200vit_debug_set(key, 0) == -1, key


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", tmp_path / "nope.so")
    with pytest.raises(_lib.B200VitError, match="no fallback"):
        _lib.lib()


def test_library_contains_hopper_instructions():
    """SASS evidence that the GEMM and the attention are wgmma code fed by TMA through mbarriers."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump) or not _lib.LIB_PATH.exists():
        pytest.skip("cuobjdump or library not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_lib.LIB_PATH)], capture_output=True, text=True).stdout
    assert "arch = sm_90a" in sass
    for mnemonic in ("HGMMA.64x256x16.F32.BF16", "HGMMA.64x128x16.F32.BF16", "HGMMA.64x64x16.F32.BF16", "UTMALDG",
                     "SYNCS"):
        assert mnemonic in sass, mnemonic
    assert "HMMA.16816" not in sass          # no warp-level mma.sync tensor path
