"""The online kernels at D = 9..16 without a device: the wide launchers dispatch exactly the D that
tests/test_gpu_online_wide.py tests, the D <= 8 launchers hand every other D to them, and the C ABI rejects what it
must (D = 17 as unsupported; a bad block or lambda at D = 9 as invalid, not as unsupported)."""
import ctypes
import os
import re

import pytest

import test_gpu_online_wide as gpu
from test_kernel_instances_cpu import _cases, _function, _src

DISCO_ERR_INVALID, DISCO_ERR_UNSUPPORTED = -1, -2


def test_wide_dispatch_sets():
    assert set(gpu.WIDE_D) == _cases(_function(_src("online_wide.cu"), "cudaError_t launch_scm_recursive_wide("),
                                      "launch_recursive_wide_d")
    assert set(gpu.WIDE_D) == _cases(_function(_src("online.cu"), "cudaError_t launch_filter_sum_blocks_wide("),
                                     "launch_filter_d")


def test_narrow_launchers_fall_through_to_the_wide_ones():
    src = _src("online.cu")
    for narrow, wide in (("launch_scm_recursive", "launch_scm_recursive_wide"),
                         ("launch_filter_sum_blocks", "launch_filter_sum_blocks_wide")):
        body = _function(src, "cudaError_t %s(" % narrow)
        assert re.search(r"default\s*:\s*return\s+%s\(a,\s*st\)" % wide, body), narrow


def test_engine_constants_match_the_launcher():
    body = _function(_src("online_wide.cu"), "static cudaError_t launch_recursive_wide_d(")
    m = re.search(r"constexpr int TS = (\d+), NS = (\d+);", body)
    assert m and (int(m.group(1)), int(m.group(2))) == (gpu.TS, gpu.NS)


def test_build_compiles_online_wide():
    from disco_b200 import build
    assert "online_wide.cu" in build.SOURCES and os.path.exists(os.path.join(build.CSRC, "online_wide.cu"))


@pytest.fixture(scope="module")
def lib():
    from disco_b200 import build, _lib
    build.build()
    return _lib.load()


def test_abi_rejects_before_any_launch(lib):
    p = ctypes.c_void_p(16)          # never dereferenced: every call below fails validation first
    rec, filt = lib.disco_scm_recursive, lib.disco_filter_sum_blocks
    #          Y  Z  mask R0s R0n Rss Rnn lambda block pow n_utt K  C  T   n_fft sel n_sel
    assert rec(p, p, p, None, None, p, p, 0.9, 8, 2, 1, 2, 16, 30, 512, None, 0, None) == DISCO_ERR_UNSUPPORTED
    assert rec(p, None, p, None, None, p, p, 0.9, 8, 2, 1, 1, 17, 30, 512, None, 0, None) == DISCO_ERR_UNSUPPORTED
    #           W  conj Y  Z  out resid ref block lag n_utt K  C  T   n_fft sel n_sel
    assert filt(p, 1, p, p, p, p, 0, 8, 1, 1, 9, 9, 30, 512, None, 0, None) == DISCO_ERR_UNSUPPORTED
    # D = 9 (8 nodes x 2 mics, and one array of 9): accepted shapes, bad parameters -> invalid
    for K, C in ((8, 2), (1, 9)):
        for block in (0, 65):
            assert rec(p, p, p, None, None, p, p, 0.9, block, 2, 1, K, C, 30, 512, None, 0, None) == DISCO_ERR_INVALID
            assert b"block" in lib.disco_last_error()
            assert filt(p, 1, p, p, p, p, 0, block, 1, 1, K, C, 30, 512, None, 0, None) == DISCO_ERR_INVALID
        assert rec(p, p, p, None, None, p, p, 1.0, 8, 2, 1, K, C, 30, 512, None, 0, None) == DISCO_ERR_INVALID
        assert b"lambda" in lib.disco_last_error()
        assert filt(p, 1, p, p, p, p, 9, 8, 1, 1, K, C, 30, 512, None, 0, None) == DISCO_ERR_INVALID   # ref = D
