"""The C-ABI library loads on a CPU-only box and exports every symbol include/b200_tetris_mcts.h declares; compute
entry points fail loudly (no CPU fallback).  No compute call is made here."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    from tetris_mcts_b200 import build
    return build.build()


def test_header_symbols_exported(built):
    from tetris_mcts_b200 import _lib
    names = _lib.exported_symbols()
    assert len(names) >= 25
    L = C.CDLL(built)
    missing = [n for n in names if not hasattr(L, n)]
    assert not missing, missing
    nm = subprocess.run(["nm", "-D", "--defined-only", built], capture_output=True, text=True).stdout
    for n in names:
        assert re.search(r"\bT %s\b" % n, nm), n


def test_sm90a_code_present(built):
    out = subprocess.run(["cuobjdump", "-lelf", built], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out[:300]


def test_no_cpu_fallback(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the loud-failure path is for CPU-only boxes")
    from tetris_mcts_b200 import _lib
    from tetris_mcts_b200.engine import BatchedEngine
    with pytest.raises(_lib.B200Error) as ei:
        BatchedEngine(4, max_nodes=64, eval_kind="synthetic")
    assert ei.value.code == 2 and "no CUDA device" in str(ei.value)
    from tetris_mcts_b200.pyTetris import Tetris
    with pytest.raises(_lib.B200Error):
        Tetris((20, 10), 1, 0, 0)


def test_product_never_imports_oracle():
    """oracle/ is test infrastructure: nothing under tetris_mcts_b200/ may import, load or exec it."""
    pkg = os.path.join(ROOT, "tetris_mcts_b200")
    for d, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(d, f), errors="ignore").read()
                assert "oracle_py" not in txt and "liboracle" not in txt and "import oracle" not in txt, os.path.join(d, f)


def test_config_struct_layout_matches_header():
    from tetris_mcts_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "b200_tetris_mcts.h")).read()
    body = hdr[hdr.index("typedef struct {"):hdr.index("} b200_config;")]
    fields = []
    for decl in re.findall(r"(?:int32_t|uint32_t|double)\s+([^;]+);", body):
        fields += [f.strip() for f in decl.split(",")]
    assert fields == [f[0] for f in _lib.Config._fields_]
