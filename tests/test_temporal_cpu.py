"""The temporal-metric oracle (oracle/temporal_oracle.py) against the outputs of the unmodified reference
(tests/golden/temporal.npz): bit for bit, and each mutation of the oracle's arithmetic changes at least one bit."""
import numpy as np
import pytest

import temporal_cases as tc
from oracle import temporal_oracle as to


def test_rebuilt_inputs_are_the_ones_the_reference_ran_on():
    z = tc.fixture()
    got = tc.input_digests()
    assert got == {k[len("digest_"):]: str(z[k]) for k in z if k.startswith("digest_")}


def _smoothing_matches(z, **mutation):
    """[case index]: whether the (mutated) oracle gives the reference's bits."""
    xs = tc.smoothing_inputs()
    return [tc.digest(to.one_euro(xs[k], mc, b, **mutation)) == str(z[f"sm{i}_digest"])
            for i, (k, mc, b) in enumerate(tc.smoothing_cases())]


def test_oracle_smoothing_matches_reference_bitwise():
    z = tc.fixture()
    ok = _smoothing_matches(z)
    assert len(ok) > 100 and all(ok), [i for i, o in enumerate(ok) if not o]


def _nonuniform_matches(z, dt, tag, **mutation):
    x, t = tc.nonuniform_case(dt)
    return tc.digest(to.one_euro(x, 0.004, 0.7, t=t, **mutation)) == str(z[f"ou_{tag}_digest"])


def test_oracle_nonuniform_times_match_reference_bitwise():
    z = tc.fixture()
    assert _nonuniform_matches(z, np.float32, "f32") and _nonuniform_matches(z, np.float64, "f64")


def test_nan_and_inf_stay_in_their_channel():
    for x in tc.smoothing_inputs():
        bad = ~np.isfinite(x.reshape(len(x), -1))
        if bad.any():
            for mc, b in tc.PAIRS:
                flat = to.one_euro(x, mc, b).reshape(len(x), -1)
                ch = bad.any(0)
                for c in np.flatnonzero(ch):   # NaN from the bad frame on (an inf gives a = inf / inf)
                    assert np.isnan(flat[np.argmax(bad[:, c]):, c]).all()
                assert np.isfinite(flat[:, ~ch]).all()


def _accel_matches(z, **mutation):
    out = []
    for i, gt, pred, v, vis in tc.accel_cases():
        per_window, valid = to.accel_error(gt, pred, vis, **mutation)
        out.append(tc.digest(per_window[valid]) == str(z[f"ac{i}_{v}_digest"]))
    return out


def test_oracle_accel_matches_reference_bitwise():
    z = tc.fixture()
    assert all(_accel_matches(z))
    # the joint mean is pinned for every joint count in the fixture
    assert {gt.shape[1] for _, gt, *_ in tc.accel_cases()} == {14, 17, 24}


@pytest.mark.parametrize("mutation", ["fma", "weights_swapped", "cutoff_2pi_in_double", "beta_on_raw_dx"])
def test_smoothing_mutation_changes_fixture_bits(mutation):
    assert not all(_smoothing_matches(tc.fixture(), **{mutation: True}))


def test_unit_te_mutation_changes_nonuniform_case():
    z = tc.fixture()
    assert not _nonuniform_matches(z, np.float32, "f32", unit_te=True)
    assert not _nonuniform_matches(z, np.float64, "f64", unit_te=True)


@pytest.mark.parametrize("mutation", ["vis_first_frame_only", "naive_mean"])
def test_accel_mutation_changes_fixture_bits(mutation):
    assert not all(_accel_matches(tc.fixture(), **{mutation: True}))


def test_video_loop_agrees_with_reference_block():
    z = tc.fixture()
    pred_j3d, gt_j3d, masks = tc.video_set()
    for smooth, tag in ((True, "smooth"), (False, "raw")):
        accel, mpjpe, pa, acc_t, mpjpe_t, pa_t = to.evaluate_video_f64(pred_j3d, gt_j3d, list(masks), smooth)
        np.testing.assert_allclose(accel, z[f"vid_{tag}_accel"], rtol=1e-5)
        np.testing.assert_allclose(mpjpe, z[f"vid_{tag}_mpjpe"], rtol=1e-5)
        np.testing.assert_allclose(mpjpe_t, z[f"vid_{tag}_mpjpe_total"], rtol=1e-5)
        np.testing.assert_allclose(pa_t, z[f"vid_{tag}_pa_total"], rtol=1e-5)
        assert np.isnan(acc_t) and np.isnan(z[f"vid_{tag}_accel_total"])   # the 1- and 2-frame videos have none
        if smooth:
            scale = np.abs(gt_j3d[np.concatenate([np.flatnonzero(m) for m in masks])]).max(axis=(1, 2))
            assert (np.abs(pa - z["vid_smooth_pa"]) <= 1e-6 * scale[:, None]).all()
