"""CPU oracle for the disco MWF beamforming path — TEST INFRASTRUCTURE ONLY.

Nothing in ``disco_b200`` (the product) may import from this package.  Allowed
importers: ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs, and there only as the checker or
the CPU baseline — never as the thing shipped or measured as the GPU path.

Contents
--------
librosa_np   NumPy restatement of the librosa (<=0.9) STFT / iSTFT semantics the
             reference calls (librosa itself is a third-party dependency that is
             absent here and unpinned in the reference's requirements.txt).
tango_np     Loop-faithful NumPy/SciPy restatement of the reference algorithm
             (tango.py:252-457, internal_formulas.py:31-103, dnn/utils.py:44-71,
             sigproc_utils.py:12-55), keeping the reference's dtype flow
             (complex64 SCM, single-precision LAPACK cggev, complex128 filters).
tango_f64    Vectorised float64 evaluation of the same mathematics ("truth" for
             error budgeting; also a much faster CPU baseline).
ref_shim     Imports the UNMODIFIED reference from /root/reference (only where it
             is mounted) through sys.modules stubs for its absent third-party
             imports; used by make_golden.py to pin the restatement.
make_golden  Generates tests/golden/*.npz by running the real reference.
lfilter_np   scipy.signal.lfilter's direct form II transposed restated one ufunc
             per operation, bit-equal to scipy; the yardstick of band_stats.

Parity pinning status: the reference ships no golden vectors for this path
(SURVEY.md §4).  The MWF mathematics (SCM, intern_filter, filter-and-sum, the
two-step exchange) IS pinned: tests/golden/ holds outputs of the reference's own
``offline_tango`` / ``intern_filter`` executed in the authoring container through
ref_shim.  The STFT/iSTFT boundary is "parity unpinned" in the strict sense:
librosa is absent, so its semantics are restated (librosa_np) and cross-checked
against torch.stft/istft and scipy.signal.get_window only.
"""
