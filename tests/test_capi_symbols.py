"""CPU: libdt_b200.so builds, loads, and exports every symbol include/dt_b200.h
declares; the ctypes table covers the header; product code never imports oracle/."""
import ctypes
import os
import re

import pytest

from detectandtrack_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, 'include', 'dt_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(dt_[a-z0-9_]+)\s*\(', src)))


def test_library_loads_and_exports_all_header_symbols():
    names = _header_functions()
    assert len(names) >= 8
    lib = ctypes.CDLL(_lib.LIB_PATH)
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_ctypes_table_matches_header():
    names = set(_header_functions())
    table = set(_lib.SIGNATURES) | set(_lib.HOST_FUNCS) | {'dt_last_error'}
    assert names == table, (names - table, table - names)


def test_abi_version_and_error_channel():
    lib = _lib.lib()
    assert lib.dt_abi_version() == 4
    # argument validation happens on the host before any CUDA call: usable without a GPU
    rc = lib.dt_bbox_overlaps(None, 4, 4, None, 4, 4, 99, None, 4, None)
    assert rc != 0
    assert b'T=99' in lib.dt_last_error()
    with pytest.raises(RuntimeError, match='T=99'):
        _lib.check(rc, 'dt_bbox_overlaps')


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, 'detectandtrack_b200')
    bad = []
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                txt = open(os.path.join(dp, f)).read()
                if re.search(r'^\s*(from|import)\s+oracle\b', txt, flags=re.M) or 'oracle/_ref' in txt and f.endswith('.py'):
                    bad.append(os.path.join(dp, f))
    for f in ['tools/' + n for n in sorted(os.listdir(os.path.join(ROOT, 'tools'))) if n.endswith('.py')]:
        p = os.path.join(ROOT, f)
        if os.path.exists(p) and re.search(r'^\s*(from|import)\s+oracle\b', open(p).read(), flags=re.M):
            bad.append(p)
    assert not bad, bad


def test_ops_fail_loudly_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip('CUDA present')
    import numpy as np
    from detectandtrack_b200.core import nms_wrapper
    with pytest.raises(RuntimeError):
        nms_wrapper.nms(np.zeros((3, 5), np.float32), 0.5)
