"""oracle/inputs_oracle.py, the float64 restatement of the training inputs' device rule, against the unmodified
reference's statistics in tests/golden/inputs.npz (CPU only).

Every comparison of distributions runs on fixed seeds, so its p-value is a fixed number: a test fails when it is below
P_FAIL (1e-4), and the smallest p-value seen is printed so that a margin shrinking towards the threshold shows."""
import numpy as np
import pytest

from inputs_cases import CASES, GOLDEN, P_FAIL, SEEDS, case, error_table, fixture_pvalues, ordered_table
from oracle import demo_oracle as do
from oracle import inputs_oracle as io

M = int(GOLDEN["M"])


@pytest.mark.parametrize("name", CASES)
def test_oracle_samples_match_reference_fixture(name):
    """M samples of each case, per joint: the outcome annuli with their radial bins (and, where the sources overlap,
    the 2-D offsets) have the reference's distribution."""
    assert M >= 5000
    joints, area, _ = case(name)
    out = io.synthesize_pose(np.repeat(joints[None], M, 0), np.full(M, area), SEEDS)
    ps = fixture_pvalues(name, out)
    p, where = min(ps)
    print(f"{name}: smallest p = {p:.3g} ({where}) over {len(ps)} tests")
    assert p > P_FAIL, (p, where)


def test_phase_two_takes_inv_from_the_partners_synthesized_row():
    """Joints 2, 4, .., 16 use their partner's output row as the inv source, (0, 0) when it was zeroed (still gated by
    the partner's ORIGINAL visibility); joints 1, 3, .., 15 use the partner's original coordinate."""
    joints, area, _ = case("all_visible")
    B = 64
    trace = {}
    out = io.synthesize_pose(np.repeat(joints[None], B, 0), np.full(B, area), SEEDS, trace=trace)
    for j in range(1, 17):
        assert trace[f"has_inv_{j}"].all()
        want = out[:, j - 1, :2] if j % 2 == 0 else np.broadcast_to(joints[j + 1, :2], (B, 2))
        np.testing.assert_array_equal(trace[f"inv_{j}"], want)
    np.testing.assert_array_equal(trace["has_inv_0"], False)
    # area 0 and joints 1, 2 on one point: every candidate of joint 1 is absent, so it is zeroed and joint 2's inv
    # source is (0, 0)
    z = joints.copy()
    z[2, :2] = z[1, :2]
    trace = {}
    out = io.synthesize_pose(z[None], np.zeros(1), SEEDS, trace=trace)
    np.testing.assert_array_equal(out[0, 1], 0.0)
    assert trace["has_inv_2"][0]
    np.testing.assert_array_equal(trace["inv_2"][0], 0.0)
    np.testing.assert_array_equal(out[0, 2], [z[2, 0], z[2, 1], 1.0])
    # an invisible partner is no source, whatever its coordinate
    z = joints.copy()
    z[6, 2] = 0
    trace = {}
    io.synthesize_pose(z[None], np.full(1, area), SEEDS, trace=trace)
    assert not trace["has_inv_5"][0] and trace["has_inv_6"][0]


def test_sample_rows_depend_only_on_the_sample_its_index_and_the_seed():
    rng = np.random.default_rng(3)
    B = 7
    joints = np.concatenate([rng.uniform(20, 260, (B, 17, 2)), (rng.uniform(size=(B, 17, 1)) > 0.3)], 2)
    joints = joints.astype(np.float32).astype(np.float64)
    area = rng.uniform(500, 20000, B)
    full = io.synthesize_pose(joints, area, SEEDS)
    for i in range(B):
        alone = io.synthesize_pose(joints[i:i + 1], area[i:i + 1], SEEDS, sample_index=[i])
        np.testing.assert_array_equal(alone[0], full[i])
    other = io.synthesize_pose(joints[::-1].copy(), area[::-1].copy(), SEEDS, sample_index=np.arange(B)[::-1])
    np.testing.assert_array_equal(other[::-1], full)
    assert not np.array_equal(io.synthesize_pose(joints, area, (SEEDS[0] + 1, SEEDS[1])), full)
    assert not np.array_equal(io.synthesize_pose(joints, area, (SEEDS[0], SEEDS[1] + 1)), full)


def test_embedded_sigmas_equal_the_reference():
    np.testing.assert_array_equal(np.array(io.KPS_SIGMAS_X10) / 10.0, GOLDEN["kps_sigmas"])
    src = open(io.__file__.replace("oracle/inputs_oracle.py", "pose2mesh_release_b200/csrc/inputs.cu")).read()
    body = src[src.index("KPS_SIGMAS_X10[N_KPS] = {") + 25:]
    device = [float(v) for v in body[:body.index("}")].replace("\n", " ").split(",")]
    np.testing.assert_array_equal(np.array(device) / 10.0, GOLDEN["kps_sigmas"])


def test_error_model_validates_the_table():
    from pose2mesh_release_b200.inputs import Human36MErrorModel

    table, names = error_table()
    m = Human36MErrorModel(table, names)
    assert m.joint_names == tuple(names)
    mean, std, weight = ordered_table()
    for i in range(17):
        assert tuple(m.table[i].mean) == tuple(mean[i]) and m.table[i].weight == weight[i]

    def broken(i, **kw):
        t = [dict(e) for e in table]
        t[i].update(kw)
        return t

    bad = [
        (table[:-1], names),                                   # an entry missing
        (table + [dict(table[0])], names),                     # a duplicate entry
        (table, names[:-1]),                                   # 16 names
        (broken(3, mean=(float("nan"), 0.0)), names),
        (broken(3, std=(1.0, -0.5)), names),
        (broken(3, std=(1.0, float("inf"))), names),
        (broken(3, weight=1.5), names),
        (broken(3, weight=-0.1), names),
        (broken(3, mean=(1.0,)), names),
        ([{k: v for k, v in e.items() if k != "weight"} for e in table], names),
    ]
    for t, n in bad:
        with pytest.raises(ValueError):
            Human36MErrorModel(t, n)


def test_h36m_oracle_draws_follow_the_table_and_the_reference():
    """10^5 fixed-seed samples per joint: kept fraction within 5 sigma of the weight; mean and std of the kept values
    within 5 sigma of the table; and the kept fraction and mean within 5 sigma of the reference's restated draws."""
    mean, std, weight = ordered_table()
    n = 100_000
    noise = io.generate_syn_error((mean, std, weight), n, SEEDS).astype(np.float64)
    kept = (noise != 0).any(axis=2)
    Mr = int(GOLDEN["h36m_M"])
    for i in range(17):
        k = kept[:, i].sum()
        frac, w = k / n, float(np.float32(weight[i]))
        assert abs(frac - w) <= 5 * max(np.sqrt(w * (1 - w) / n), 1 / n), (i, frac, w)
        v = noise[kept[:, i], i]
        for c in range(2):
            assert abs(v[:, c].mean() - mean[i, c]) <= 5 * std[i, c] / np.sqrt(k), (i, c)
            assert abs(v[:, c].std() - std[i, c]) <= 5 * std[i, c] / np.sqrt(2 * k), (i, c)
        kr = int(GOLDEN["h36m_kept"][i])
        fr = kr / Mr
        sd = np.sqrt(max(w * (1 - w), 1 / n) * (1 / n + 1 / Mr))
        assert abs(frac - fr) <= 5 * sd + 1e-12, (i, frac, fr)
        mr = GOLDEN["h36m_sum"][i] / kr
        for c in range(2):
            assert abs(v[:, c].mean() - mr[c]) <= 5 * std[i, c] * np.sqrt(1 / k + 1 / kr), (i, c)


def test_noise_free_crop_is_the_demo_normalisation():
    """The crop the noise is added in is k_normalize_pose2d's: without noise the oracle's pipeline is the demo's."""
    rng = np.random.default_rng(5)
    poses = rng.uniform(50, 900, (6, 19, 2)).astype(np.float32)
    got, _ = io.training_pose2d(poses, "none")
    want = np.stack([do.normalize_pose2d(p.astype(np.float64)) for p in poses])
    np.testing.assert_allclose(got, want, atol=1e-5)
    # the area of the tight box in the crop: the reference maps its corners through the affine transform
    m = io.crop_map(poses)
    for b in range(len(poses)):
        tight = do.get_bbox(poses[b])
        trans = do.affine_from_bbox(do.process_bbox(tight.copy()), (io.INPUT_SHAPE[1], io.INPUT_SHAPE[0]))
        xmin, ymin, xmax, ymax = tight[0], tight[1], tight[0] + tight[2], tight[1] + tight[3]
        p1, p2, p3 = (trans @ np.array([x, y, 1.0]) for x, y in ((xmin, ymin), (xmax, ymin), (xmax, ymax)))
        area = np.hypot(*(p2 - p1)) * np.hypot(*(p3 - p2))
        np.testing.assert_allclose(io.crop_area(m, "tight")[b], area, rtol=1e-6)  # float32 corner points
