"""online_tango's evaluation inputs without a device: the ops call sites of the helpers it calls for them are covered
by tests/test_gpu_online_eval.py, its argument errors are raised before any device work, and the float64
split-statistics step of oracle/online_split_np reduces to online_mwf."""
import numpy as np
import pytest
import torch

import test_gpu_online_eval as ev
import test_gpu_tango_routes as routes


def test_every_eval_call_site_is_covered():
    """Each `ops.<name>(` call in the evaluation helpers of online.py (the rule of test_gpu_tango_routes.call_sites)
    is named by a row of the GPU test's table, every row names a site the sources have, and every row's test exists."""
    sites = ev.eval_sites()
    assert sites, "no call sites parsed"
    missing = set(sites) - set(ev.SITES)
    assert not missing, "ops call sites no row of test_gpu_online_eval.SITES reaches: %s" % sorted(missing)
    unknown = set(ev.SITES) - set(sites)
    assert not unknown, "the table names call sites the sources do not have: %s" % sorted(unknown)
    for site, test in ev.SITES.items():
        assert callable(getattr(ev, test, None)), (site, test)
    # the helpers are not among the functions whose sites the route table covers
    assert not set(ev.EVAL_FUNCS) & set(routes.SITE_FUNCS["online.py"])


def _cpu_inputs():
    y = torch.zeros(1, 2, 2, 2048)
    m = torch.zeros(1, 2, 9, 257)
    return y, m


@pytest.mark.parametrize("kwargs,exc", [
    (dict(), ValueError),                                                       # no masks and no s / n
    (dict(s="s"), ValueError),                                                  # s without n
    (dict(masks="m", mask_for_z="compressed"), ValueError),
    (dict(masks="m", mask_for_z="use_oracle_refs"), ValueError),
    (dict(masks="m", mask_for_z="use_oracle_zs"), ValueError),
    (dict(masks="m", s="s", mask_for_z="use_oracle_zs"), ValueError),          # n missing
    (dict(masks="m", mask_for_z=None), TypeError),
    (dict(s="s", n="n", mask_for_z=None), TypeError),
    (dict(s="s", n="n", vads=("crnn", "irm1")), ValueError),
    (dict(s="s", n="n", vads=("irm1", "rnn")), ValueError),
    (dict(s="s", n="n", vads=("irm1", "xyz1")), ValueError),
    (dict(s="s", n="n", mask_for_z="use_oracle_sigs"), NotImplementedError),
    (dict(masks="m", mask_for_z="use_oracle_sigs"), NotImplementedError),
], ids=lambda v: v.__name__ if isinstance(v, type) else "-".join("%s=%s" % kv for kv in sorted(v.items())))
def test_online_tango_rejects_before_device_work(kwargs, exc):
    """The errors of tango_batched, raised from CPU tensors: no device call has been made when they are."""
    from disco_b200 import online, tango
    y, m = _cpu_inputs()
    kw = {k: {"m": (m, m), "s": y, "n": y}.get(v, v) if isinstance(v, str) and k in ("masks", "s", "n") else v
          for k, v in kwargs.items()}
    with pytest.raises(exc) as on:
        online.online_tango(y, **kw)
    # the same error as tango_batched for the same arguments
    with pytest.raises(exc) as off:
        tango.tango_batched(y, kw.get("s"), kw.get("n"), masks=kw.get("masks"), vads=kw.get("vads", ("irm1", "irm1")),
                            mask_for_z=kw.get("mask_for_z", "local"))
    assert str(on.value) == str(off.value)


@pytest.mark.parametrize("D,lag,R0", [(3, 1, False), (3, 0, True), (9, 2, True), (9, 1, False)])
def test_split_oracle_reduces_to_online_mwf(D, lag, R0):
    """online_mwf_split(X, m X, (1 - m) X) == online_mwf(X, m, power=2) to 1e-12: z, W and both matrix sequences."""
    from oracle import online_np, online_split_np, solve_f64, tango_np
    rng = np.random.default_rng(10 * D + lag)
    F, T, block = 5, 6 * D + 3, 4
    X = rng.standard_normal((D, F, T)) + 1j * rng.standard_normal((D, F, T))
    m = rng.uniform(0.05, 0.95, size=(F, T))
    r0 = None
    if R0:
        A = rng.standard_normal((2, F, D, D)) + 1j * rng.standard_normal((2, F, D, D))
        r0 = tuple(0.1 * a @ a.conj().swapaxes(-1, -2) for a in A)
    scm = tango_np.spatial_correlation_matrix
    solve = lambda Rs, Rn, mu, ft, r: solve_f64.solve(Rs, Rn, mu, ft, r)
    kw = dict(lambda_cor=0.9, block=block, lag=lag, mu=1.0, rank=1, ref=D - 1, R0=r0)
    a = online_np.online_mwf(X, m, scm, solve, power=2, **kw)
    b = online_split_np.online_mwf_split(X, m * X, (1 - m) * X, scm, solve, **kw)
    for x, w in zip(b, a):
        assert np.linalg.norm(x - w) <= 1e-12 * np.linalg.norm(w)
    # the speech and noise stacks are read where they are meant to be: swapping them changes the filters
    c = online_split_np.online_mwf_split(X, (1 - m) * X, m * X, scm, solve, **kw)
    assert np.linalg.norm(c[1] - a[1]) > 1e-3 * np.linalg.norm(a[1])
