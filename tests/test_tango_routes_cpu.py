"""Tango's route layer without a device: the two float64 restatements agree at non-default options, and the route
table of tests/test_gpu_tango_routes.py covers every `ops` call site of tango.py / online.py.

The reference pins only ref_mic = 0 and mu = 1, gevd, rank 1 (its tango.py hard-codes them, and for ref_mics != 0 it
reads mask_z before node 0 has one).  What the project means by the other options is stated twice, independently:
oracle/tango_np.py (the reference's loops, LAPACK zggev in double precision) and oracle/tango_f64.py (vectorised, a
Cholesky-whitened eigh).  Their agreement to 1e-9 is what pins those options; the GPU route tests use them as truth."""
import numpy as np
import pytest

import test_gpu_tango_routes as routes
from conftest import rel_l2

NAMES = ("yf", "sf", "nf", "z_y", "z_s", "z_n", "zn", "masks_z", "mask_w")


def _f64_solve(Rss, Rnn, mu, filter_type, rank):
    """tango_f64's closed forms, its GEVD without the 1e-12 diagonal loading (tango_np solves the unloaded pencil;
    the loading alone moves a rank-2 filter of these inputs by 2e-9)."""
    from oracle import tango_f64
    if filter_type == "gevd":
        return tango_f64.gevd_filter(Rss, Rnn, mu, rank, loading=0.0)[0]
    return tango_f64.solve(Rss, Rnn, mu, filter_type, rank)


@pytest.mark.parametrize("mfz", ["local", "distant"])
@pytest.mark.parametrize("fi", range(len(routes.FILTERS)), ids=["%s-r%s-mu%g" % f for f in routes.FILTERS])
@pytest.mark.parametrize("ref", ["0", "last"])
@pytest.mark.parametrize("K,C", [(1, 3), (3, 2)])
def test_yardsticks_agree_at_every_option(K, C, ref, fi, mfz):
    """tango_f64 == tango_np(double=True, granularity='bin') to 1e-9 complex relative L2 on all nine outputs, with the
    step-1 mask of microphone ref_mic, the step-2 mask of microphone 0 and zn = Y[ref_mic] - z_y."""
    from disco_b200.synth import make_batch
    from oracle import tango_f64, tango_np
    typ, rank, mu = routes.FILTERS[fi]
    ref_mic = 0 if ref == "0" else C - 1
    y, s, n = (a[0] for a in make_batch(1, K, C, 3000, seed0=10 * K + C))
    kw = dict(n_fft=256, n_hop=128, mu=mu, filter_type=typ, rank=rank, mask_for_z=mfz, ref_mic=ref_mic)
    a = tango_f64.offline_tango(y, s, n, solve=_f64_solve, **kw)
    b = dict(zip(NAMES, tango_np.offline_tango(y, s, n, granularity="bin", double=True, **kw)))
    for nm in NAMES:
        for k in range(K):
            e = rel_l2(a[nm][k], b[nm][k])
            assert e <= 1e-9, (nm, k, e)
    # the options are not inert here: the neighbouring reference microphone changes masks_z and zn
    other = tango_f64.offline_tango(y, s, n, solve=_f64_solve, **dict(kw, ref_mic=C - 1 - ref_mic))
    assert rel_l2(other["zn"][0], a["zn"][0]) > 1e-3 and rel_l2(other["masks_z"][0], a["masks_z"][0]) > 1e-3
    if ref_mic != 0:
        assert not np.array_equal(a["masks_z"], a["mask_w"])           # step 2 keeps microphone 0


def _named():
    out = set()
    for r in routes.ROUTES + routes.ONLINE:
        out.update(r["calls"])
    return out


def test_every_call_site_has_a_route():
    """Each `ops.<name>(` call in tango_batched, tango_step1, tango_step2, _z_for_stats, _offline_tango_ragged,
    online_mwf and online_tango is one the table's rows must reach (or one listed as reached elsewhere)."""
    sites = routes.call_sites()
    named = _named()
    assert not set(routes.EXEMPT) & named, "a site listed as covered elsewhere is also named by a row"
    missing = set(sites) - named - set(routes.EXEMPT)
    assert not missing, "ops call sites no ROUTES / ONLINE row reaches: %s" % sorted(missing)
    unknown = (named | set(routes.EXEMPT)) - set(sites)
    for r in routes.ROUTES:
        unknown |= set(r["never"]) - set(sites)
    assert not unknown, "the table names call sites the sources do not have: %s" % sorted(unknown)
    for r in routes.ROUTES:
        assert not set(r["calls"]) & set(r["never"]), r["id"]


# the rows of the route table, by the inputs that select each route
REQUIRED = {
    "fuse_dual": {("dual_c1", 1, 1, 256), ("dual_c4_512", 1, 4, 512), ("dual_c3", 1, 3, 256),
                  ("dual_c4_eqvad_last", 1, 4, 256)},
    "same_mask": {("same_c4", 1, 4, 512), ("same_c6", 1, 6, 512), ("same_c10", 1, 10, 256)},
    "fuse_mid": {("mid_c6_512", 1, 6, 512), ("mid_c3_1024", 1, 3, 1024), ("mid_c7_1024", 1, 7, 1024)},
    "k1_generic": {("k1_generic_c12", 1, 12, 256)},
    "fuse_multi": {("multi_c2k3", 3, 2, 256), ("multi_c1k4", 4, 1, 512), ("multi_c4k2", 2, 4, 1024)},
    "k_generic": {("kgen_c5k2", 2, 5, 512), ("kgen_c2k5", 5, 2, 256)},
    "exchange": {("x_distant", 3, 2, 256), ("x_compressed", 3, 2, 256), ("x_oracle_refs", 3, 2, 256),
                 ("x_oracle_zs", 3, 2, 256), ("x_previous", 3, 2, 256)},
    "estimator": {("est_k1c4", 1, 4, 512), ("est_k3c2", 3, 2, 256)},
    "ragged": {("ragged_local", 3, 3, 256), ("ragged_compressed", 3, 3, 256)},
}


def test_route_table_rows():
    have = {}
    for r in routes.ROUTES:
        have.setdefault(r["route"], set()).add((r["id"], r["K"], r["C"], r["n_fft"]))
    for route, rows in REQUIRED.items():
        assert rows <= have.get(route, set()), (route, sorted(rows - have.get(route, set())))
    modes = {r["mfz"] for r in routes.ROUTES if r["route"] == "exchange"}
    assert modes == {"distant", "compressed", "use_oracle_refs", "use_oracle_zs", "previous"}
    eq = [r for r in routes.ROUTES if r["id"] == "dual_c4_eqvad_last"][0]
    assert eq["vads"][0] == eq["vads"][1] and eq["masks"] == "oracle" and eq["ref"] == "last"


def test_every_route_sees_every_option():
    """Over the table expanded by filter setting, every route runs ref_mic 0 and C - 1 (the ragged adapter has no
    ref_mic), oracle and external masks, and both output layouts as the one compared with float64."""
    seen = {}
    for r in routes.ROUTES:
        for fi in range(len(routes.FILTERS)):
            typ, rank, mu, ref, kind, layout = routes.case_options(r, fi)
            d = seen.setdefault(r["route"], {"ref": set(), "masks": set(), "layout": set(), "filters": set()})
            if r["C"] > 1:
                d["ref"].add("0" if ref == 0 else ("last" if ref == r["C"] - 1 else "mid"))
            if kind == "callable":
                kind = ("oracle", "external")[fi % 2]
            d["masks"].add({"same": "external"}.get(kind, kind))
            d["layout"].add(layout)
            d["filters"].add((typ, rank, mu))
    for route, d in seen.items():
        if route != "ragged":
            assert d["ref"] == {"0", "last"}, (route, d["ref"])
        assert d["masks"] == {"oracle", "external"}, (route, d["masks"])
        assert d["layout"] == {"FT", "TF"}, (route, d["layout"])
        assert d["filters"] == set(routes.FILTERS), route


def test_online_rows():
    rows = routes.ONLINE
    assert {(r["K"], r["C"]) for r in rows} >= {(1, 4), (2, 3), (1, 12), (4, 6)}
    assert {r["ref"] for r in rows} == {0, "last"} and {r["rank"] for r in rows} == {1, 2}
    assert {r["lag"] for r in rows} == {0, 1, 2} and {r["block"] for r in rows} == {4, 16}
    assert {r["R0"] for r in rows} == {True, False} and {r["n_fft"] for r in rows} == {256, 512, 1024}
    # R0 with a single node (seeds both steps) and with several (step 2 from zeros)
    assert {r["K"] == 1 for r in rows if r["R0"]} == {True, False}
