"""SASS of the GEMM instances compiled for the encoder layer's flag sets (gemm_bf16_kernel's EPI parameter): every
TMA-store instance has them, and their epilogues -- from the tile's last HGMMA to its first UTMASTG -- carry no
per-pair branches (QKV, FC1) and no activation code (out-proj, FC2)."""
import functools
import os
import re
import shutil
import subprocess

import pytest

from vit_pytorch_b200 import _lib

QKV, FC1 = 1 | 8, 1 | 2 | 8               # EPI_BIAS | EPI_LNFOLD (| EPI_GELU)
RES_STATS, RES_STATS_BIAS = 4 | 16, 1 | 4 | 16  # EPI_RESIDUAL | EPI_STATS (| EPI_BIAS)
# BLOCK_N, STAGES, PATCH, RES, TMA_OUT, SIG, EPI
NAME = re.compile(r"gemm_bf16_kernelILi(\d+)ELi(\d+)ELb([01])ELb([01])ELb([01])ELb([01])ELi(n?\d+)E")


@functools.lru_cache(maxsize=None)
def _sass():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump) or not _lib.LIB_PATH.exists():
        return None
    return subprocess.run([cuobjdump, "-sass", str(_lib.LIB_PATH)], capture_output=True, text=True).stdout


def _kernels():
    sass = _sass()
    if sass is None:
        pytest.skip("cuobjdump or library not available")
    out = {}
    for fn in re.split(r"\n\s*Function : ", sass)[1:]:
        m = NAME.search(fn.split("\n", 1)[0])
        if not m:
            continue
        block_n, _, _, res, tma_out, _, epi = m.groups()
        ops = re.findall(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", fn)
        out[(int(block_n), res == "1", tma_out == "1", int(epi.replace("n", "-")))] = ops
    return out


def _epilogue(ops):
    last = max(i for i, op in enumerate(ops) if op.startswith("HGMMA"))
    first_store = next(i for i in range(last, len(ops)) if ops[i].startswith("UTMASTG"))
    return ops[last:first_store]


def test_encoder_flag_sets_have_their_own_instances():
    k = _kernels()
    for block_n in (128, 256):
        for epi in (QKV, FC1):
            assert (block_n, False, True, epi) in k, (block_n, epi)
        for epi in (RES_STATS, RES_STATS_BIAS):
            assert (block_n, True, True, epi) in k, (block_n, epi)


def test_compiled_epilogues_are_straight_line():
    k = _kernels()
    for (block_n, res, tma_out, epi), ops in k.items():
        if epi < 0:
            continue
        epilogue = _epilogue(ops)
        if res:
            # the per-pair bounds tests stay (a slab's columns past N are stale), the activations are compiled out
            assert not any(op.startswith("MUFU") for op in epilogue), (block_n, epi)
        else:
            # a few reconvergence regions per tile (the vector-buffer wait, the LN-fold statistics), none per pair
            bssy = sum(op.startswith("BSSY") for op in epilogue)
            assert bssy <= 8, (block_n, epi, bssy)
    # the generic instance of the same shape still branches per pair
    generic = _epilogue(k[(256, False, True, -1)])
    assert sum(op.startswith("BSSY") for op in generic) > 32
