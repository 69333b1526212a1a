"""Per-hypothesis float64 checks of the device RANSAC (csrc/ransac.cu) that need no unique rotation, so they hold on every sample it
scores, rank-deficient ones included; and the input families that make such samples common.  Shared by test_gpu_ransac.py,
test_gpu_ransac_samples.py and test_ransac_samples_host.py.

A hypothesis draws three candidates (a_j, b_j), j = 0, 1, 2 (float32 values, exact in double), and the device solves the unscaled
Umeyama in double: am = fl(fl(fl(a0 + a1) + a2) / 3), x_j = fl(a_j - am), H' = the fma sum of x_j y_j^T, R = kabsch_rotation(H'),
t = b' - R am.  The exact sample has a-bar, alpha_j = a_j - a-bar (b-bar, beta_j likewise) and H = sum_j alpha_j beta_j^T, computed
here in long double (2^-11 of double's roundoff).  u = 2^-53, eps = 2^-52, gamma(n) = n u / (1 - n u).

Pre-solver error.  |am - a-bar| <= da = gamma(3) sum_j |a_j| / 3 per coordinate.  x_j = (alpha_j - (am - a-bar)) (1 + theta_j),
|theta_j| <= u.  The common shift cancels in the bilinear sum, because sum_j beta_j = 0 exactly: sum_j (am - a-bar) beta_j^T = 0.
What is left of x_j y_j^T - alpha_j beta_j^T, entry (r, c), plus the three-term fma sum, is at most
    E_rc = sum_j [ u (|alpha_jr| + da_r) |beta_jc| + u (|beta_jc| + db_c) |alpha_jr| + ea_jr eb_jc
                   + gamma(3) (|alpha_jr| + ea_jr) (|beta_jc| + eb_jc) ],     ea_jr = da_r + u (|alpha_jr| + da_r)  (eb alike).
The mean errors enter only through products with a rounding, so a sample far from the origin (offset 1e4) is not penalised for
its offset: every term scales with S = sum_j |alpha_j| |beta_j| except for u * da terms, second order in u.

Rotation.  R R^T = I and det R = 1 to 16 eps: R = w1 u1^T + w2 u2^T + (w1 x w2)(u1 x u2)^T of unit vectors orthogonal to a few
eps each (Gram-Schmidt, or any_perpendicular on a rank-1 H).

Optimal value, not optimal argument.  A 3-point H has rank <= 2 (the alpha_j sum to 0), so max over rotations of tr(R H) =
sigma_1 + sigma_2 for every sample; on rank-1 H every R with R u1 = v1 attains it, and R need not be unique.  The device's gap
    sigma_1 + sigma_2 - tr(R H) <= [max tr(. H') - tr(R H')] + [sigma_1 + sigma_2 - max tr(. H')] + |tr(R (H' - H))|.
The second and third terms are at most sum E each (|R_ij| <= 1; the exact optimum R* is a candidate for H').  The first is the
solver's suboptimality on H' in value, a backward error: the rank-1 branch gives up at most 2 sigma_2' <= 2 sqrt(3.2e-30)
sigma_1' = 16.1 eps sigma_1' (svd3.cuh's threshold), and the 24 Jacobi plane rotations, the normalisations and R's products move
the value by a few eps sigma_1' each, 48 eps in all: C_VALUE = 64, with sigma_1' <= |H'|_F <= S + sum E.  The long-double H is
rounded to double for kabsch_ld's singular values, which moves sigma_1 + sigma_2 by at most 2 u sum |H|.
    value_bound = C_VALUE eps (S + sum E) + 3 sum E + 2 u sum |H|.
Nothing divides by a singular gap: the bound holds on rank-1 and zero H.  A wrong reflection loses 2 sigma_2 or more, a rotation
that loses u1 -> v1 by an angle phi loses about sigma_1 phi^2 / 2 (phi = 1e-6 already exceeds the bound), and a rank-1 branch
taken at sigma_2 / sigma_1 = 1e-13 (a rank threshold of 1e-24) loses up to sigma_2 = 1e-13 sigma_1, about 6x the bound.

Translation.  t_r = fl(b'_r - fma(R_r0, am_0, fma(R_r1, am_1, R_r2 am_2))) against b-bar_r - (R a-bar)_r:
    |t - (b-bar - R a-bar)|_r <= db_r + sum_k |R_rk| da_k + gamma(4) (sum_k |R_rk| |am_k| + |b'_r|).
A sample whose three a_j (or three b_j) are one point has am = a exactly (fl(fl(2a) + a) = 3a and 3a / 3 = a for float32 a), H' = 0,
R = I and t = fl(b' - am), bit for bit.

Scores.  d^2 = |R p + t - q|^2 over the candidates, on the device and here alike in double: each coordinate of R p + t is a
three-fma chain, within gamma(4) (sum_k |R_rk p_k| + |t_r| + |q_r|) = del_r of exact after the subtraction of q, and the squares'
fma sum is within gamma(3) of its terms, so |d^2' - d^2| <= derr = sum_r (2 |e_r| del_r + del_r^2) + gamma(3) sum_r (|e_r| + del_r)^2.
Two such evaluations differ by 2 derr: a candidate with |d^2 - r * r| <= 2 derr is ambiguous, every other is decided (r * r is
the device's double product).  good lies between the sure inliers and the sure inliers plus the ambiguous ones.  Where none is
ambiguous the inliers are known and sum d^2 is within 2 (sum derr + gamma(good) sum d^2) of the device's ordered sum, so
    |rmse' - rmse| <= 1e-12 rmse + that / (good (rmse' + rmse)) + 2 u rmse.
"""
import numpy as np

from float64_bounds import EPS64, U64, gamma64, kabsch_ld
from oracle import ransac_oracle as O

LD = np.longdouble
C_VALUE = 64.0
ORTHO = 16.0 * EPS64
LD_REL = 2.0 ** -60            # long double arithmetic: 2^-64 per operation, a few operations deep
DEGENERATE = 1e-9              # sigma_2 / sigma_1 at or below which a sample's rotation is not determined to float accuracy
WORST = {}                     # worst error / bound of each check over the session


def note(what, err, bound):
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0.0))
    r = float(np.max(r, initial=0.0))
    WORST[what] = max(WORST.get(what, 0.0), r)
    return r


def report():
    return ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items()))


def device_mean(x):
    """[I,3,3] -> [I,3]: the device's fl(fl(fl(x0 + x1) + x2) / 3) (numpy float64 rounds each operation alike)."""
    return ((x[:, 0] + x[:, 1]) + x[:, 2]) / 3.0


def samples(p, q, idx):
    """The exact samples of draws idx [I,3] over candidates p, q [M,3] (float32 values).  Rows with a non-finite coordinate are
    flagged (finite = False) and carry zeros."""
    a, b = p[idx], q[idx]                                            # [I, j, 3]
    finite = np.isfinite(a).all((1, 2)) & np.isfinite(b).all((1, 2))
    a = np.where(finite[:, None, None], a, 0.0)
    b = np.where(finite[:, None, None], b, 0.0)
    al, bl = a.astype(LD), b.astype(LD)
    abar, bbar = al.sum(1) / 3, bl.sum(1) / 3
    alpha, beta = al - abar[:, None], bl - bbar[:, None]
    H = np.einsum("ijr,ijc->irc", alpha, beta)
    aa, ab = np.abs(alpha).astype(np.float64), np.abs(beta).astype(np.float64)
    da = gamma64(3) * np.abs(a).sum(1) / 3
    db = gamma64(3) * np.abs(b).sum(1) / 3
    ea = da[:, None] + U64 * (aa + da[:, None])
    eb = db[:, None] + U64 * (ab + db[:, None])
    E = (np.einsum("ijr,ijc->irc", U64 * (aa + da[:, None]), ab) + np.einsum("ijr,ijc->irc", aa, U64 * (ab + db[:, None]))
         + np.einsum("ijr,ijc->irc", ea, eb) + gamma64(3) * np.einsum("ijr,ijc->irc", aa + ea, ab + eb)
         + LD_REL * np.einsum("ijr,ijc->irc", aa, ab))
    S = (np.sqrt((aa * aa).sum(2)) * np.sqrt((ab * ab).sum(2))).sum(1)
    return dict(a=a, b=b, finite=finite, abar=abar, bbar=bbar, H=H, E=E, S=S, da=da, db=db, am=device_mean(a), bm=device_mean(b),
                one_a=(a == a[:, :1]).all((1, 2)), one_b=(b == b[:, :1]).all((1, 2)))


def sigma(H):
    """Singular values [I,3] of long-double H (kabsch_ld on H rounded to double); exact zeros for H = 0."""
    s = kabsch_ld(np.asarray(H, np.float64))[1]
    return np.where((np.asarray(H) == 0).all((1, 2))[:, None], 0.0, s)


def value_bound(sm):
    sumE = sm["E"].sum((1, 2))
    return C_VALUE * EPS64 * (sm["S"] + sumE) + 3.0 * sumE + 2.0 * U64 * np.abs(sm["H"]).sum((1, 2)).astype(np.float64)


def value_gap(R, sm, s=None):
    """sigma_1 + sigma_2 - tr(R H) per sample (long double tr, R [I,3,3] double)."""
    s = sigma(sm["H"]) if s is None else s
    tr = np.einsum("irc,icr->i", np.asarray(R, np.float64).astype(LD), sm["H"]).astype(np.float64)
    return s[:, 0] + s[:, 1] - tr


def translation_bound(R, sm):
    Ra = np.abs(R)
    return sm["db"] + np.einsum("irk,ik->ir", Ra, sm["da"]) + gamma64(4) * (np.einsum("irk,ik->ir", Ra, np.abs(sm["am"]))
                                                                            + np.abs(sm["bm"])) + LD_REL * (
        np.abs(sm["bbar"]).astype(np.float64) + np.einsum("irk,ik->ir", Ra, np.abs(sm["abar"]).astype(np.float64)))


def recount(R, t, p, q, r2):
    """float64 d^2 of every candidate under (R [3,3], t [3]) and its evaluation error bound derr (module header)."""
    with np.errstate(invalid="ignore", over="ignore"):
        e = p @ R.T + t - q
        d2 = (e * e).sum(1)
        dl = gamma64(4) * (np.abs(p) @ np.abs(R).T + np.abs(t) + np.abs(q))
        ae = np.abs(e)
        derr = (2 * ae * dl + dl * dl).sum(1) + gamma64(3) * ((ae + dl) ** 2).sum(1)
        ok = np.isfinite(d2) & np.isfinite(derr)
        band = 2.0 * derr
        sure_in = ok & (d2 + band < r2)
        amb = ok & ~sure_in & (d2 - band < r2)
    return d2, derr, sure_in, amb


def check_set(dev, b, src, tgt, labels, r, max_iteration=5000, seed=O.DEFAULT_SEED, rows=slice(None)):
    """Every hypothesis of device set b (dev: `ransac_packed(..., info=True, hypotheses=True)` as numpy) against the float64 checks
    of the module header, and its selection, T and labels against its own keys and transform.  src, tgt [N,3] float32 and labels
    [N] are the set's rows; rows selects them in dev['labels'].  Returns {'draws', 'M', 'ratio' [I], 'best'}."""
    src64 = np.asarray(src, np.float32).astype(np.float64)
    tgt64 = np.asarray(tgt, np.float32).astype(np.float64)
    cand = O.candidates(labels)
    M, I, r2 = len(cand), int(max_iteration), float(r) * float(r)
    good, rmse = dev["hyp_good"][b], dev["hyp_rmse"][b]
    T = dev["hyp_trans"][b].reshape(I, 3, 4)
    out_labels = dev["labels"][rows]
    assert out_labels.shape == (len(src64),)
    assert not out_labels[np.setdiff1d(np.arange(len(src64)), cand)].any(), "a row that is not a candidate was labelled"
    eye = np.zeros((3, 4))
    eye[:, :3] = np.eye(3)
    if M < 3:
        assert int(dev["status"][b]) == 1 and not good.any() and not rmse.any() and (T == eye).all()
        assert int(dev["best_iteration"][b]) == -1 and not out_labels.any()
        assert np.array_equal(dev["trans"][b], np.eye(4, dtype=np.float32))
        return {"draws": np.zeros((0, 3), np.int64), "M": M, "ratio": np.zeros(0), "best": -1}
    p, q = src64[cand], tgt64[cand]
    idx = O.draws(seed, I, M)
    sm = samples(p, q, idx)
    fin = sm["finite"]
    R, t = T[:, :, :3], T[:, :, 3]
    # samples with a non-finite coordinate: good = 0, [I | 0]
    assert not good[~fin].any() and not rmse[~fin].any() and (T[~fin] == eye).all()
    # rotation
    RL = R[fin].astype(LD)
    orth = np.abs(np.einsum("irk,ick->irc", RL, RL) - np.eye(3, dtype=LD)).max((1, 2)).astype(np.float64)
    det = np.abs(np.linalg.det(R[fin]) - 1.0)
    assert np.isfinite(R[fin]).all() and (orth <= ORTHO).all() and (det <= ORTHO).all(), (float(orth.max()), float(det.max()))
    note("rotation", np.maximum(orth, det), np.full(orth.shape, ORTHO))
    # H = 0 (three a_j or three b_j one point): R = I and t = fl(b' - am) bit for bit
    zero = fin & (sm["one_a"] | sm["one_b"])
    assert (R[zero] == np.eye(3)).all() and (t[zero] == sm["bm"][zero] - sm["am"][zero]).all()
    # optimal value
    s = np.zeros((I, 3))
    s[fin] = sigma(sm["H"][fin])
    fs = {k: (v[fin] if isinstance(v, np.ndarray) and v.shape[:1] == (I,) else v) for k, v in sm.items()}
    gap, vb = value_gap(R[fin], fs, s[fin]), value_bound(fs)
    bad = np.flatnonzero(np.abs(gap) > vb)
    assert not len(bad), ("value gap", np.flatnonzero(fin)[bad[:6]], gap[bad[:6]], vb[bad[:6]], s[fin][bad[:6]])
    note("value", np.abs(gap), vb)
    # translation
    te = np.abs(t[fin] - (fs["bbar"] - np.einsum("irk,ik->ir", R[fin].astype(LD), fs["abar"]))).astype(np.float64)
    tb = translation_bound(R[fin], fs)
    assert (te <= tb).all(), ("translation", float((te / tb).max()))
    note("translation", te, tb)
    # scores of the device's own transforms
    for i in np.flatnonzero(fin):
        d2, derr, sure_in, amb = recount(R[i], t[i], p, q, r2)
        lo, na = int(sure_in.sum()), int(amb.sum())
        assert lo <= int(good[i]) <= lo + na, (i, int(good[i]), lo, na)
        if na == 0:
            g = lo
            if g == 0:
                assert rmse[i] == 0.0, i
                continue
            S = float(d2[sure_in].sum())
            dS = 2.0 * (float(derr[sure_in].sum()) + gamma64(g) * S)
            ref = np.sqrt(S / g)
            den = g * (float(rmse[i]) + ref)
            tol = 1e-12 * ref + (dS / den if den > 0 else np.sqrt(dS / g)) + 2 * U64 * ref
            err = abs(float(rmse[i]) - ref)
            assert err <= tol, (i, float(rmse[i]), ref, tol)
            note("rmse", np.array([err]), np.array([tol]))
    # the winner: the open3d rule on the device's own keys; T and labels are its own transform's
    best = int(dev["best_iteration"][b])
    assert best == O.select(good, rmse)
    if best < 0:
        assert int(dev["status"][b]) == 2 and not out_labels.any() and np.array_equal(dev["trans"][b], np.eye(4, dtype=np.float32))
        assert float(dev["fitness"][b]) == 0.0 and float(dev["inlier_rmse"][b]) == 0.0
    else:
        assert int(dev["status"][b]) == 0
        want = np.eye(4, dtype=np.float32)
        want[:3] = T[best].astype(np.float32)
        assert np.array_equal(dev["trans"][b], want)
        assert float(dev["fitness"][b]) == good[best] / M and float(dev["inlier_rmse"][b]) == float(rmse[best])
        _, _, sure_in, amb = recount(R[best], t[best], p, q, r2)
        lab = out_labels[cand]
        assert set(np.unique(lab).tolist()) <= {0.0, 1.0}
        assert np.array_equal(lab[~amb], sure_in[~amb].astype(np.float32)) and int(lab.sum()) == int(good[best])
    ratio = np.where(s[:, 0] > 0, s[:, 1] / np.where(s[:, 0] > 0, s[:, 0], 1.0), np.inf)
    return {"draws": idx, "M": M, "ratio": np.where(fin, ratio, np.nan), "best": best}


# ---------------------------------------------------------------------------------------------------
# input families: (src [N,3] float32, tgt [N,3] float32, labels [N] float32) sets
# ---------------------------------------------------------------------------------------------------
def exact_motion(x, k=0):
    """An exact float32 rigid motion: a signed axis permutation plus a dyadic translation (no rounding, so a family keeps its
    rank and ratio in the target cloud too)."""
    perms = [((1, -1), (0, 1), (2, 1)), ((2, 1), (1, -1), (0, -1)), ((0, 1), (1, 1), (2, 1))]
    y = np.empty_like(x)
    for i, (src_axis, sgn) in enumerate(perms[k % 3]):
        y[:, i] = sgn * x[:, src_axis]
    return (y + np.float32([0.5, -0.25, 0.125])).astype(np.float32)


def small_m_sets(M, preset, count=12, seed=0):
    """count sets of M candidates from synthetic pairs, inlier fractions 1/4 .. 1, with two non-candidate rows each."""
    from pointdsc_b200.synth import make_pair
    out = []
    for k in range(count):
        frac = (1, 2, 3, 4)[k % 4] / 4
        pr = make_pair(1000 * M + 17 * k + seed, 4 * M + 8, preset, 0.5)
        s, t = pr["src_keypts"].numpy(), pr["tgt_keypts"].numpy()
        n_in = max(1, int(round(frac * M)))
        n_half = (4 * M + 8) // 2
        rows = np.concatenate([np.arange(n_in), n_half + np.arange(M - n_in), [n_half - 1, len(s) - 1]])
        lab = np.ones(M + 2, np.float32)
        lab[-2:] = 0.0
        out.append((s[rows].copy(), t[rows].copy(), lab))
    return out


def duplicate_sets(seed=0):
    """many sources onto one target; one source onto many targets; repeated identical correspondences."""
    from pointdsc_b200.synth import make_pair
    pr = make_pair(seed, 60, "3dmatch", 0.6)
    s, t = pr["src_keypts"].numpy(), pr["tgt_keypts"].numpy()
    lab = np.ones(60, np.float32)
    many_to_one = (s.copy(), t[(np.arange(60) // 5) * 5].copy(), lab)
    one_to_many = (s[(np.arange(60) // 4) * 4].copy(), t.copy(), lab)
    rep = np.repeat(np.arange(12), 5)
    repeated = (s[rep].copy(), t[rep].copy(), lab)
    return {"many_to_one": many_to_one, "one_to_many": one_to_many, "repeated": repeated}


def collinear_set(offset, m=24, axis=1):
    """m candidates on one line along `axis` (the other two coordinates equal in every row), centred at `offset` * (1, 1, 1);
    targets are an exact motion of the sources (plus one off-line outlier pair)."""
    x = np.full((m, 3), offset, np.float32)
    x[:, axis] = (offset + np.linspace(-1.0, 1.0, m)).astype(np.float32)
    y = exact_motion(x, 0)
    x = np.concatenate([x, np.float32([[offset + 0.5, offset - 0.5, offset + 0.25]])])
    y = np.concatenate([y, np.float32([[offset, offset + 3.0, offset]])])
    return x, y, np.ones(m + 1, np.float32)


def near_collinear_triple(ratio, L=1.0):
    """Three candidates along y with the middle one lifted along z by eps: sum alpha alpha^T = diag(0, 2 L^2, 2 eps^2 / 3), so
    sigma_2 / sigma_1 = eps^2 / (3 L^2) (eps rounded to float32: the family's actual ratio is measured, not assumed).  The x
    coordinate is kept off 0 so that any_perpendicular (which starts from the x axis) picks a u2 orthogonal to the true one."""
    eps = np.float32(L * np.sqrt(3.0 * ratio))
    x = np.float32([[0.25, -L, 0.0], [0.25, 0.0, eps], [0.25, L, 0.0]])
    return x, exact_motion(x, 1), np.ones(3, np.float32)


NEAR_RATIOS = (1e-6, 1e-10, 1e-13, 1e-15)


def point_sets(seed=3):
    """all targets one point; all sources one point (H = 0 for every sample)."""
    g = np.random.default_rng(seed)
    x = (g.random((20, 3)) * 2.0).astype(np.float32)
    one = np.tile(np.float32([[0.3, -1.7, 2.9]]), (20, 1))
    return {"targets_one_point": (x, one.copy(), np.ones(20, np.float32)),
            "sources_one_point": (one.copy(), x, np.ones(20, np.float32))}
