"""CPU guards of the extent model (tests/abi_extents.py) and of the negative matrix of tests/test_gpu_ops_extents.py:
a row for every pointer parameter of every entry point include/disco_b200.h declares, a negative-matrix entry for
every wrapper that hands a tensor to the library, and the model's own verdicts on fake registrations."""
import ast
import os

import pytest

import abi_extents as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_model_covers_every_header_pointer_parameter():
    hp = M.header_params()
    assert len(hp) >= 40
    missing = [(n, p) for n, ps in hp.items() for p in M.pointer_params(ps) if p not in M.ROWS.get(n, {})]
    assert not missing, missing
    stale = [(n, p) for n, row in M.ROWS.items() for p in row if p not in {q for _, q in hp.get(n, ())}]
    assert not stale, stale
    for n, row in M.ROWS.items():
        for p, (mode, dtype, count) in row.items():
            assert mode in ("r", "w", "rw", "host") and dtype in M.ITEMSIZE, (n, p)
            assert callable(count) or count[0] in ("stft", "bss", "stoi"), (n, p)


def _wrappers_passing_tensors():
    """Every @_on_device function of ops.py that hands a tensor to _ptr."""
    tree = ast.parse(open(os.path.join(ROOT, "disco_b200", "ops.py")).read())
    out = set()
    for fn in tree.body:
        if not isinstance(fn, ast.FunctionDef):
            continue
        if not any(isinstance(d, ast.Name) and d.id == "_on_device" for d in fn.decorator_list):
            continue
        if any(isinstance(c, ast.Call) and isinstance(c.func, ast.Name) and c.func.id == "_ptr" and c.args
               for c in ast.walk(fn)):
            out.add(fn.name)
    return out


def test_negative_matrix_covers_every_wrapper():
    import test_gpu_ops_extents as G
    wrappers = _wrappers_passing_tensors()
    assert len(wrappers) >= 25
    assert wrappers == set(G._TENSOR_ARGS), wrappers ^ set(G._TENSOR_ARGS)
    assert set(G.SPECIFIC) == wrappers
    for op in wrappers:
        ids = [cid for cid, _ in G.negative_cases(op)]
        for arg in G._TENSOR_ARGS[op]:
            assert any(cid.startswith(arg + ":") for cid in ids), (op, arg)
    # spectra ops: wrong F for n_fft; workspace consumers: every workspace mismatch
    for op in ("masked_scm", "filter_sum_scm", "tango_mid", "filter_sum", "filter_dual", "scm_recursive",
               "filter_sum_blocks", "istft", "istft_lengths", "stream_istft", "stream_istft_slots"):
        assert "F129_for_n_fft512" in [cid for cid, _ in G.negative_cases(op)], op
    for op in ("mwf_solve_workspace", "mwf_solve_workspace2", "scm_from_workspace"):
        ids = [cid for cid, _ in G.negative_cases(op)]
        for want in ("ws:one_slot_short", "ws:G+1", "ws:other_mask_sets", "ws:reserved_sms", "ws:dtype", "ws:cpu"):
            assert want in ids, (op, want)


class FakeSizes:
    """The fused kernel's workspace as csrc/api.cu sizes it (stft_ws_bytes), for a fixed number of slots per group."""

    def __init__(self, slots):
        self.slots = slots

    def stft_ws(self, n_grp, C, length, n_fft, n_set):
        return n_grp * self.slots * n_set * 2 * C * C * (n_fft // 2 + 1) * 4

    def bss_ws(self, *a):
        return 0

    def stoi_ws(self, *a):
        return 0


def _check(name, args, spans, sizes=FakeSizes(3)):
    reg = {}
    for k, (nbytes, dtype) in spans.items():
        addr = 0x10000 * (len(reg) + 1)
        reg[addr] = M.Span(addr, nbytes, dtype, 0)
        args[k] = addr
    M.check_call(name, args, reg.get, sizes, 0, lambda v: (len(v), "i32"))


def _masked_scm(T, F_Y):
    n_utt, K, C, n_fft = 2, 1, 4, 512
    D = C + K - 1
    a = dict(n_utt=n_utt, K=K, C=C, T=T, n_fft=n_fft, node_sel=0, n_sel=0, Z=0, mask=0)
    spans = {"Y": (n_utt * C * T * F_Y * 8, "c64"), "Rss": (n_utt * F_Y * D * D * 8, "c64"),
             "Rnn": (n_utt * F_Y * D * D * 8, "c64")}
    return a, spans


def test_model_rejects_129_bins_at_n_fft_512():
    a, spans = _masked_scm(10, 257)
    _check("disco_masked_scm", a, spans)                     # consistent: accepted
    a, spans = _masked_scm(10, 129)
    with pytest.raises(M.Refused, match="Y reads past the end"):
        _check("disco_masked_scm", a, spans)


def test_model_rejects_rnn_shorter_than_rss():
    n_mat, D = 514, 4
    a = dict(n_mat=n_mat, D=D, T1=0)
    full = (n_mat * D * D * 8, "c64")
    _check("disco_mwf_solve", dict(a), {"Rss": full, "Rnn": full, "W": (n_mat * D * 8, "c64")})
    with pytest.raises(M.Refused, match="Rnn reads past the end"):
        _check("disco_mwf_solve", dict(a), {"Rss": full, "Rnn": ((n_mat - 1) * D * D * 8, "c64"),
                                            "W": (n_mat * D * 8, "c64")})
    with pytest.raises(M.Refused, match="Rnn is f32"):
        _check("disco_mwf_solve", dict(a), {"Rss": full, "Rnn": (n_mat * D * D * 8, "f32"),
                                            "W": (n_mat * D * 8, "c64")})


def test_model_rejects_workspace_one_slot_short():
    G, C, L, n_fft = 3, 4, 16000, 512
    F = n_fft // 2 + 1
    sizes = FakeSizes(5)
    need = sizes.stft_ws(G, C, L, n_fft, 2)
    slot = 2 * 2 * C * C * F * 4
    a = dict(n_grp=G, C=C, length=L, n_fft=n_fft)
    out = {"W": (2 * G * F * C * 8, "c64"), "T1": (2 * G * F * C * 8, "c64")}
    _check("disco_mwf_solve_workspace2", dict(a), dict(out, workspace=(need, "f32")), sizes)
    with pytest.raises(M.Refused, match="workspace reads past the end"):
        _check("disco_mwf_solve_workspace2", dict(a), dict(out, workspace=(need - slot, "f32")), sizes)
    # a workspace read as one set of a two-set one is in extent; a larger plan (more slots) is not
    _check("disco_scm_from_workspace", dict(a, n_set=1, set=0),
           {"workspace": (need, "f32"), "Rss": (G * F * C * C * 8, "c64"), "Rnn": (G * F * C * C * 8, "c64")}, sizes)
    with pytest.raises(M.Refused, match="workspace reads past the end"):
        _check("disco_mwf_solve_workspace2", dict(a), dict(out, workspace=(need, "f32")), FakeSizes(6))


def test_model_checks_host_arrays_and_devices():
    import ctypes
    n_utt, K, C, T, n_fft = 2, 3, 2, 10, 256
    F, D = 129, 4
    sel = (ctypes.c_int * 2)(0, 2)
    a = dict(n_utt=n_utt, K=K, C=C, T=T, n_fft=n_fft, node_sel=sel, n_sel=2, mask=0, R0ss=0, R0nn=0, block=4)
    spans = {"Y": (n_utt * 2 * C * T * F * 8, "c64"), "Z": (n_utt * K * T * F * 8, "c64"),
             "Rss": (n_utt * 2 * 3 * F * D * D * 8, "c64"), "Rnn": (n_utt * 2 * 3 * F * D * D * 8, "c64")}
    _check("disco_scm_recursive", dict(a), dict(spans))
    with pytest.raises(M.Refused, match="node_sel holds 3"):
        _check("disco_scm_recursive", dict(a, node_sel=(ctypes.c_int * 3)(0, 1, 2)), dict(spans))
    reg = {0x1000: M.Span(0x1000, 1 << 20, "c64", 1)}
    with pytest.raises(M.Refused, match="lives on cuda:1"):
        M.check_call("disco_transpose_c64", dict(batch=1, rows=2, cols=2, out=0, **{"in": 0x1000}), reg.get,
                     FakeSizes(1), 0, None)
