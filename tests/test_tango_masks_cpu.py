"""The mask and geometry decisions of the Python orchestration, checked without a GPU: which compressed signals
feed a step-2 mask estimator, which mask types exist, and how Y / Z / node_sel map onto a concatenated-channel
launch (disco_b200/ops.py)."""
import numpy as np
import pytest

from disco_b200 import ops
from disco_b200.compat.tango import get_z_for_mask
from disco_b200.tango import _mask_kind, _z_for_mask


@pytest.mark.parametrize("z_sigs", ["zs_hat", "zn_hat", "interleaved"])
@pytest.mark.parametrize("K", [2, 3, 4, 5])
def test_z_for_mask_matches_get_z_for_mask(K, z_sigs):
    # signal t of node j is the plane filled with 100 * t + j, so the reference's selection names its sources
    z_s = [np.full((3, 2), j, np.float32) for j in range(K)]
    z_n = [np.full((3, 2), 100 + j, np.float32) for j in range(K)]
    for k in range(K):
        ref = [int(p[0, 0]) for p in get_z_for_mask(z_s, z_n, k, K, z_sigs)]
        assert [100 * t + j for t, j in _z_for_mask(k, K, z_sigs)] == ref


@pytest.mark.parametrize("vad, kind", [("irm1", "oracle"), ("ibm2", "oracle"), ("iam1", "oracle"), ("irm9", "oracle"),
                                       ("ivad", "ivad"), ("crnn", "dnn"), ("rnn", "dnn")])
def test_mask_kind_accepts_the_reference_types(vad, kind):
    assert _mask_kind(vad) == kind


@pytest.mark.parametrize("vad", ["foo1", "irm", "irmx", "irm12", "ibm", "vad", "cnn", "crnn1", "", None, 1])
def test_mask_kind_rejects_anything_else(vad):
    with pytest.raises(ValueError):
        _mask_kind(vad)


B, C, T, F = 2, 3, 47, 257


def test_cat_geometry_without_z():
    # no exchange: every (b, k) is its own single-node problem
    assert ops._cat_geometry((B, 4, C, T, F)) == (B * 4, 1, None, 1, 0)


@pytest.mark.parametrize("z_layout, flag", [("BK", 0), ("KB", 1)])
def test_cat_geometry_all_nodes_and_selection(z_layout, flag):
    K = 4
    z = (B, K, T, F) if z_layout == "BK" else (K, B, T, F)
    assert ops._cat_geometry((B, K, C, T, F), z, None, z_layout) == (B, K, None, K, flag)
    n_utt, k, sel, n_sel, zl = ops._cat_geometry((B, 2, C, T, F), z, [1, 3], z_layout)
    assert (n_utt, k, list(sel), n_sel, zl) == (B, K, [1, 3], 2, flag)


@pytest.mark.parametrize("z_layout", ["BK", "KB"])
@pytest.mark.parametrize("axis", ["B", "T", "F"])
def test_cat_geometry_rejects_a_z_that_differs_from_y(z_layout, axis):
    K = 3
    dims = dict(B=B, T=T, F=F)
    dims[axis] += 1 if axis != "T" else -1
    z = (dims["B"], K, dims["T"], dims["F"]) if z_layout == "BK" else (K, dims["B"], dims["T"], dims["F"])
    with pytest.raises(ValueError):
        ops._cat_geometry((B, K, C, T, F), z, None, z_layout)
    with pytest.raises(ValueError):
        ops._cat_geometry((B, 1, C, T, F), z, [0], z_layout)


def test_cat_geometry_rejects_other_z_ranks_and_layouts():
    for z in [(B, 3, T), (B, 3, 1, T, F)]:
        with pytest.raises(ValueError):
            ops._cat_geometry((B, 3, C, T, F), z)
    with pytest.raises(ValueError):
        ops._cat_geometry((B, 3, C, T, F), (B, 3, T, F), None, "TB")


def test_cat_geometry_rejects_a_selection_that_does_not_match_y():
    z = (B, 4, T, F)
    with pytest.raises(ValueError):
        ops._cat_geometry((B, 3, C, T, F), z)                  # all 4 nodes selected, Y holds 3
    with pytest.raises(ValueError):
        ops._cat_geometry((B, 2, C, T, F), z, [0, 1, 2])
    with pytest.raises(ValueError):
        ops._cat_geometry((B, 3, C, T, F), z, [2])


def test_filter_args():
    assert ops._filter_args("gevd", 1) == (0, 1)
    assert ops._filter_args("r1-mwf", "full") == (1, 0)
    assert ops._filter_args("mwf", None) == (2, 0)
    with pytest.raises(AttributeError):                     # internal_formulas.py:79
        ops._filter_args("lcmv", 1)
