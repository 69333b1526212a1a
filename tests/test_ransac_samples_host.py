"""The per-hypothesis RANSAC checks of tests/ransac_samples.py on the CPU: each input family is what it claims to be, the bounds
accept two other float64 solvers of the same samples (the oracle's LAPACK Umeyama and a solve in another summation order), and a
rotation taken off the optimal family by a small angle, or with its second direction flipped, breaks the value bound."""
import numpy as np
import pytest

from float64_bounds import kabsch64, kabsch_ld
from oracle import ransac_oracle as O
from oracle.icp_oracle import umeyama
from ransac_samples import (DEGENERATE, NEAR_RATIOS, check_set, collinear_set, duplicate_sets, near_collinear_triple,
                            point_sets, samples, sigma, small_m_sets, translation_bound, value_bound, value_gap)

I = 400


def families():
    out = {f"small_{M}_{p}": small_m_sets(M, p, count=4) for M in (3, 5, 8) for p in ("3dmatch", "kitti")}
    out.update({k: [v] for k, v in duplicate_sets().items()})
    out.update({f"collinear_{o:g}": [collinear_set(o)] for o in (0.0, 1e2, 1e4)})
    out["near_collinear"] = [near_collinear_triple(x) for x in NEAR_RATIOS]
    out.update({k: [v] for k, v in point_sets().items()})
    return out


FAMILIES = families()


def _samples(st, I=I):
    s, t, lab = st
    c = O.candidates(lab)
    p, q = s[c].astype(np.float64), t[c].astype(np.float64)
    sm = samples(p, q, O.draws(O.DEFAULT_SEED, I, len(c)))
    return sm, sigma(sm["H"])


def test_mean_of_three_equal_float32_is_exact():
    """fl(fl(a + a) + a) / 3 == a for float32 a, which makes H = 0 and t = fl(b - a) exact on a single-index sample."""
    g = np.random.default_rng(0)
    with np.errstate(over="ignore"):
        a = (g.standard_normal(100000) * 10.0 ** g.integers(-40, 39, 100000)).astype(np.float32)
    a = np.concatenate([a, np.float32([0.0, -0.0, 1e-45, -1e-45, 1.17549435e-38, 3.4028235e38, -3.4028235e38, 1e4, 1e-4])])
    a = a[np.isfinite(a)].astype(np.float64)
    assert len(a) > 90000
    assert np.array_equal(((a + a) + a) / 3.0, a)


def test_constructions():
    # collinear: every sample has rank <= 1, so sigma_2 = 0 up to the long double's rounding
    for o in (0.0, 1e2, 1e4):
        for axis in (0, 1, 2):
            s, t, lab = collinear_set(o, axis=axis)
            c = O.candidates(lab)[:-1]                                    # the line, without the outlier pair
            x = s[c].astype(np.float64)
            assert (x[:, [k for k in range(3) if k != axis]] == o).all() and len(np.unique(x[:, axis])) > 20
            sm, sg = _samples((s[:-1], t[:-1], lab[:-1]))
            assert (sg[:, 1] <= 1e-17 * sg[:, 0]).all()
    # near-collinear triples: the ratio as built, on either side of the double rank threshold sqrt(3.2e-30) = 1.79e-15
    for want in NEAR_RATIOS:
        sm, sg = _samples(near_collinear_triple(want), 60)
        full = (np.sort(O.draws(O.DEFAULT_SEED, 60, 3), 1) == [0, 1, 2]).all(1)
        ratio = sg[full, 1] / sg[full, 0]
        assert np.allclose(ratio, ratio[0], rtol=1e-6) and 0.5 * want < ratio[0] < 2 * want, (want, ratio[0])
        assert (ratio[0] > 1.79e-15) == (want > 1.79e-15)
    # all targets / all sources one point: H = 0 on every sample
    for st in point_sets().values():
        sm, sg = _samples(st)
        assert not sm["H"].any() and not sg.any() and (sm["one_a"] | sm["one_b"]).all()
    # duplicates: rank-deficient samples are common
    for name, st in duplicate_sets().items():
        sm, sg = _samples(st, 2000)
        assert (sg[:, 1] <= DEGENERATE * sg[:, 0]).mean() > 0.05, name
    # small M: fractions and M as stated
    for M in (3, 8, 32):
        for st in small_m_sets(M, "3dmatch"):
            assert len(O.candidates(st[2])) == M


def reordered_solve(a, b):
    """A float64 Umeyama in another summation order: means summed from the last point, H summed from the last point, LAPACK's
    SVD of H^T."""
    am, bm = ((a[:, 2] + a[:, 1]) + a[:, 0]) / 3.0, ((b[:, 2] + b[:, 1]) + b[:, 0]) / 3.0
    x, y = a - am[:, None], b - bm[:, None]
    H = x[:, 2, :, None] * y[:, 2, None, :] + x[:, 1, :, None] * y[:, 1, None, :] + x[:, 0, :, None] * y[:, 0, None, :]
    Rt = kabsch64(np.swapaxes(H, 1, 2))[0]          # the rotation that maps b onto a, transposed
    R = np.swapaxes(Rt, 1, 2)
    R = np.where((H == 0).all((1, 2))[:, None, None], np.eye(3), R)
    return R, bm - np.einsum("irk,ik->ir", R, am)


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_bounds_cover_other_float64_solvers(family):
    for st in FAMILIES[family]:
        sm, sg = _samples(st)
        fin = sm["finite"]
        Ru = np.stack([umeyama(a, b)[0] for a, b in zip(sm["a"], sm["b"])])
        Ro, to = reordered_solve(sm["a"], sm["b"])
        vb = value_bound(sm)
        for R in (Ru, Ro):
            gap = value_gap(R, sm, sg)
            assert (np.abs(gap[fin]) <= vb[fin]).all(), (family, float((np.abs(gap) / vb).max()))
        te = np.abs(to - (sm["bbar"] - np.einsum("irk,ik->ir", Ro.astype(np.longdouble), sm["abar"]))).astype(np.float64)
        assert (te <= translation_bound(Ro, sm)).all(), family


def _oracle_as_device(st, r, I=I):
    """The oracle's run of one set in the layout of ransac_packed(..., info=True, hypotheses=True): another float64 solver."""
    s, t, lab = st
    ref = O.ransac(s, t, lab, r, max_iteration=I)
    dev = {"status": np.array([ref["status"]]), "best_iteration": np.array([ref["best_iteration"]]),
           "fitness": np.array([ref["fitness"]]), "inlier_rmse": np.array([ref["inlier_rmse"]]),
           "trans": ref["trans"][None], "labels": ref["labels"]}
    if ref["M"] < 3:
        dev.update(hyp_good=np.zeros((1, I), np.int32), hyp_rmse=np.zeros((1, I)),
                   hyp_trans=np.tile(np.eye(3, 4).reshape(12), (1, I, 1)))
    else:
        dev.update(hyp_good=ref["good"][None], hyp_rmse=ref["rmse"][None], hyp_trans=ref["T"][:, :3, :].reshape(1, I, 12))
    return dev


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_check_set_accepts_the_oracle(family):
    """check_set applied to the float64 oracle's run passes: every check it makes of the device holds for another correct solver,
    whose rotations on rank-deficient samples differ from the device's."""
    for st in FAMILIES[family]:
        r = 0.6 if "kitti" in family else 0.10
        check_set(_oracle_as_device(st, r), 0, *st, r, max_iteration=I)


@pytest.mark.parametrize("phi", [1e-6])
def test_off_the_optimal_family_breaks_the_bound(phi):
    """A rotation about an axis orthogonal to v1 by phi loses at least sigma_1 (1 - cos phi) of value; with its second direction
    flipped (a half turn about u1) it loses 2 sigma_2.  Both exceed the bound wherever that loss does, which is on every sample
    with sigma_1 >= 1e-2 S (phi = 1e-6: 5e-13 sigma_1 against the bound's ~1.4e-14 S) and on every sample with 2 sigma_2 above
    the bound, rank-1 samples off the family included."""
    checked = flipped = 0
    for fam in ("small_5_3dmatch", "small_8_kitti", "many_to_one", "repeated", "collinear_100", "near_collinear"):
        for st in FAMILIES[fam]:
            sm, sg = _samples(st)
            ok = sm["finite"] & (sg[:, 0] > 0)
            R, _, _, U, V = kabsch_ld(np.asarray(sm["H"], np.float64))
            vb = value_bound(sm)
            assert (np.abs(value_gap(R, sm, sg))[ok] <= vb[ok]).all()
            # an axis orthogonal to v1 (the first target-side singular direction)
            v1 = V[:, :, 0]
            n = np.cross(v1, np.where(np.abs(v1[:, :1]) < 0.6, [[1.0, 0.0, 0.0]], [[0.0, 1.0, 0.0]]))
            n /= np.linalg.norm(n, axis=1, keepdims=True)
            K = np.zeros((len(n), 3, 3))
            K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -n[:, 2], n[:, 1], -n[:, 0]
            K -= np.swapaxes(K, 1, 2)
            Q = np.eye(3) + np.sin(phi) * K + (1 - np.cos(phi)) * K @ K
            loss = value_gap(Q @ R, sm, sg)
            sel = ok & (sg[:, 0] >= 1e-2 * sm["S"])
            assert sel.sum() > 0.5 * ok.sum(), fam
            assert (loss[sel] > vb[sel]).all(), (fam, float(np.min(loss[sel] / vb[sel])))
            assert (loss[sel] >= 0.99 * sg[sel, 0] * (1 - np.cos(phi))).all()
            checked += int(sel.sum())
            # a half turn about u1 in the source space keeps u1 -> v1 and flips u2, u3
            u1 = U[:, :, 0]
            F = 2 * u1[:, :, None] * u1[:, None, :] - np.eye(3)
            loss = value_gap(R @ F, sm, sg)
            sel = ok & (2 * sg[:, 1] > 2 * vb)
            assert (loss[sel] > vb[sel]).all(), fam
            flipped += int(sel.sum())
    assert checked > 500 and flipped > 100, (checked, flipped)
