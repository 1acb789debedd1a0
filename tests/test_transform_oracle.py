"""The numpy restatement of the rigid transform (tests/transform_oracle.py) against known answers and independent
formulas.  No GPU needed."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import fixtures as fx
import transform_oracle as to


def _rz(th):
    return np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])


def test_toy_fixture_known_answer():
    model, data = fx.toy_problem()
    A = np.array([[0, 0], [1, 1], [2, 2]], dtype=np.int32)
    r = to.estimate(model, data, A)
    R0 = _rz(np.pi / 8).T
    assert r["status"] == to.OK  # coplanar points: the determinant fixes the third axis
    assert np.abs(r["R"] - R0).max() <= 1e-14
    assert np.abs(r["t"] + R0 @ np.array([5.0, 3.0, 0.0])).max() <= 1e-14
    assert r["rmse"] <= 1e-14


@pytest.mark.parametrize("d", [2, 3])
def test_known_rotations(d):
    rng = np.random.default_rng(10 + d)
    for _ in range(20):
        R0, t0 = to.rotation(d, rng), rng.standard_normal(d) * 10
        a = rng.standard_normal((d, 50))
        b = R0 @ a + t0[:, None]
        r = to.estimate(a, b, None, [i * 50 + i for i in range(50)])
        assert r["status"] == to.OK
        assert np.abs(r["R"] - R0).max() <= 1e-13
        assert np.abs(r["t"] - t0).max() <= 1e-12
        assert abs(np.linalg.det(r["R"]) - 1) <= 1e-14


def test_scipy_align_vectors_3d():
    rng = np.random.default_rng(3)
    for _ in range(20):
        R0 = to.rotation(3, rng)
        a = rng.standard_normal((3, 40)) + 100.0
        b = R0 @ a + 0.05 * rng.standard_normal((3, 40))
        r = to.estimate(a, b, np.stack([np.arange(40), np.arange(40)], 1))
        x, y = a - a.mean(1, keepdims=True), b - b.mean(1, keepdims=True)
        rot, _ = Rotation.align_vectors(y.T, x.T)  # minimises sum |y_i - R x_i|^2
        assert np.abs(rot.as_matrix() - r["R"]).max() <= 1e-10


def test_atan2_closed_form_2d():
    rng = np.random.default_rng(4)
    for _ in range(20):
        a = rng.standard_normal((2, 30))
        th = rng.uniform(-np.pi, np.pi)
        b = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]) @ a + 0.1 * rng.standard_normal((2, 30))
        r = to.estimate(a, b, np.stack([np.arange(30), np.arange(30)], 1))
        x, y = a - a.mean(1, keepdims=True), b - b.mean(1, keepdims=True)
        ang = np.arctan2((x[0] * y[1] - x[1] * y[0]).sum(), (x * y).sum())
        R2 = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
        assert np.abs(R2 - r["R"]).max() <= 1e-12


def test_reflection_gives_best_proper_rotation():
    rng = np.random.default_rng(5)
    a = rng.standard_normal((3, 60)) * np.array([[3.0], [2.0], [1.0]])
    b = np.diag([1.0, 1.0, -1.0]) @ a  # mirrored: det H < 0
    r = to.estimate(a, b, np.stack([np.arange(60), np.arange(60)], 1))
    assert abs(np.linalg.det(r["R"]) - 1) <= 1e-14
    assert np.linalg.det(b @ a.T) < 0
    assert r["gap"] == pytest.approx(r["sv"][1] - r["sv"][2])
    # no proper rotation does better: compare against random ones near it
    x, y = a - a.mean(1, keepdims=True), b - b.mean(1, keepdims=True)
    best = np.sum((r["R"] @ x - y) ** 2)
    for _ in range(200):
        Q = Rotation.from_rotvec(0.05 * rng.standard_normal(3)).as_matrix() @ r["R"]
        assert np.sum((Q @ x - y) ** 2) >= best - 1e-9


def test_degenerate_cases():
    rng = np.random.default_rng(6)
    D1, D2 = rng.standard_normal((3, 5)), rng.standard_normal((3, 5))
    one = to.estimate(D1, D2, None, [7])
    assert one["status"] == to.DEGENERATE and np.array_equal(one["R"], np.eye(3)) and one["rmse"] == 0.0
    line = np.outer([1.0, 2.0, -1.0], np.arange(6.0))
    col = to.estimate(line, _rz(0.3) @ line, np.stack([np.arange(6), np.arange(6)], 1))
    assert col["status"] == to.DEGENERATE
    assert abs(np.linalg.det(col["R"]) - 1) <= 1e-14 and col["rmse"] <= 1e-14
    same = to.estimate(np.ones((3, 4)), np.zeros((3, 4)), np.stack([np.arange(4), np.arange(4)], 1))
    assert same["status"] == to.DEGENERATE and np.array_equal(same["R"], np.eye(3))
    assert np.array_equal(same["t"], -np.ones(3))
    empty = to.estimate(D1, D2, np.zeros((0, 2), np.int32), [])
    assert empty["status"] == to.EMPTY and np.array_equal(empty["T"], np.eye(4)) and empty["rmse"] == 0.0


def test_nonfinite_used_and_unused():
    rng = np.random.default_rng(7)
    D1, D2 = rng.standard_normal((3, 6)), rng.standard_normal((3, 6))
    D1[1, 5] = np.nan
    A = np.stack([np.arange(6), np.arange(6)], 1)
    used = to.estimate(D1, D2, A)
    assert used["status"] == to.NONFINITE and np.isnan(used["rmse"]) and np.isnan(used["T"][:3]).all()
    assert np.array_equal(used["T"][3], [0, 0, 0, 1])
    unused = to.estimate(D1, D2, A, [0, 1, 2, 3, 4])
    assert unused["status"] == to.OK and np.isfinite(unused["T"]).all()


def test_duplicate_rows_count_once_per_listing():
    rng = np.random.default_rng(8)
    D1, D2 = rng.standard_normal((3, 6)), rng.standard_normal((3, 6))
    A = np.stack([np.arange(6), np.arange(6)], 1)
    dup = to.estimate(D1, D2, A, [0, 1, 2, 3, 3, 3])
    expl = to.estimate(D1[:, [0, 1, 2, 3, 3, 3]], D2[:, [0, 1, 2, 3, 3, 3]], A)
    assert dup["k"] == 6 and np.allclose(dup["T"], expl["T"], atol=1e-14)
    assert not np.allclose(dup["T"], to.estimate(D1, D2, A, [0, 1, 2, 3])["T"])


def test_all_to_all_row_rule():
    rng = np.random.default_rng(9)
    D1, D2 = rng.standard_normal((2, 4)), rng.standard_normal((2, 5))
    rows = [0, 7, 13, 19]
    A = np.array([[r // 5, r % 5] for r in rows], dtype=np.int32)
    assert np.array_equal(to.estimate(D1, D2, None, rows)["T"], to.estimate(D1, D2, A)["T"])
    with pytest.raises(IndexError):
        to.estimate(D1, D2, None, [20])
