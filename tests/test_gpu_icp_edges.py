"""Device ICP (csrc/icp.cu) against oracle/icp_oracle.py at its decision edges: the radius, the kept / rejected threshold,
ties in d^2, the cell grid and its hash, the 2^21-cell limit, and rank-deficient updates.

test_gpu_icp.py only compares runs whose every decision is further than 1e-9 from its threshold.  Here the first
correspondence search is put exactly on an edge, in arithmetic that is exact on both sides:
  * dyadic float32 coordinates and an init that is a dyadic translation, so P = T src is exact in double on both sides;
  * offsets from a source to its targets of few significant bits, so d^2 is exact in double.
Exact-edge cases cannot use test_gpu_icp's margin gate, so each asserts (a) that the oracle's first-search decision is the
one the construction intends, and (b) that flipping that decision in the oracle (its `decide` hook) moves T by far more than
the parity tolerance: the comparison would see the device take the other side.  Every decision after the first update still
meets the 1e-9 margin (`late_margins`): the init is off by the dyadic translation DELTA, and the update that undoes it moves
each edge point at least |DELTA|^2 away from its threshold.

The CPU tests (unmarked) check the constructions; the GPU tests (marked) compare the device with the oracle on them."""
import numpy as np
import pytest
import torch

from oracle import icp_oracle as O

MARGIN = 1e-9
EPS64 = 2.0 ** -52
# Parity tolerance (test_gpu_icp._check): T within 2 float32 ulps per entry.  (b) asks a flipped decision to move T by at
# least FLIP_ULPS ulps, 500 times that.
FLIP_ULPS = 1000
RADII = [0.10, 0.3, 0.125, 1.0, 1e-3]
CAPS = [1, 30]               # one update (T is the first update, which the first search decides alone) and a full run


# ---------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------
def _ulps(a, b):
    def ordered(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


def _cell(x, lo, h):
    """The device's cell coordinate of x (double arithmetic, as icp.cu computes it)."""
    return np.floor((np.asarray(x, np.float64) - lo) / h)


def _exact_offset(r2f):
    """Non-negative (a, b, c) / 2^m with a^2 + b^2 + c^2 == r2f exactly in double (a three-square decomposition of r2f 4^m,
    largest a first, so the offset lies along x wherever r2f is itself a square)."""
    m = 0
    while r2f * 4.0 ** m != np.floor(r2f * 4.0 ** m):
        m += 1
    K = int(r2f * 4.0 ** m)
    for a in range(int(np.sqrt(K)), -1, -1):
        rem = K - a * a
        b = np.arange(int(np.sqrt(rem)) + 1, dtype=np.int64)
        c2 = rem - b * b
        c = np.round(np.sqrt(c2)).astype(np.int64)
        hit = np.flatnonzero((c * c == c2) & (c <= b))
        if len(hit):
            off = np.array([a, b[hit[-1]], c[hit[-1]]], np.float64) / 2.0 ** m
            assert (off * off).sum() == r2f
            return off
    raise AssertionError(r2f)


class Scene:
    """One set built from a background lattice and edge units.  Sources are given by their position at the first search,
    P0 = src + DELTA; `edges` lists (name, source row, intended row, intended keep) of the first search."""

    def __init__(self, r, origin=(0.0, 0.0, 0.0)):
        self.r, self.r2f, self.h = r, O.radius_sq(r), O.cell_side(r)
        self.u = u = 2.0 ** np.floor(np.log2(r))                        # dyadic, r / 2 < u <= r
        self.o = np.asarray(origin, np.float64)
        self.delta = np.array([0.0, u / 2, u / 4])                       # the init's translation
        self.src, self.tgt, self.edges = [], [], []
        self.spacing = np.array([8.0, 10.0, 12.0]) * u                   # >= 4 h: a lattice point reaches only its own target
        for i in range(4):
            for j in range(4):
                for k in range(4):
                    q = self.o + self.spacing * (i, j, k)
                    self.add(q, [q])
        self.slot = 0

    def add(self, p0, targets):
        """A source whose first-search position is p0, and targets; returns (source row, first target row)."""
        s = np.asarray(p0, np.float64) - self.delta
        assert (s.astype(np.float32).astype(np.float64) == s).all(), "source not exact in float32"
        for q in targets:
            assert (np.float32(q).astype(np.float64) == np.asarray(q, np.float64)).all(), "target not exact in float32"
        self.src.append(s)
        self.tgt.extend(np.asarray(q, np.float64) for q in targets)
        return len(self.src) - 1, len(self.tgt) - len(targets)

    def grid(self, x):
        """x rounded to a dyadic grid fine enough for every unit (u / 64)."""
        g = self.u / 64
        return np.round(np.asarray(x, np.float64) / g) * g

    def next_unit(self, y=None, z=None):
        """Centre of the next free unit slot: beyond the lattice along x, 16 u apart."""
        c = self.o + np.array([48.0 + 16.0 * self.slot, 15.0, 18.0]) * self.u
        self.slot += 1
        if y is not None:
            c[1] = y
        if z is not None:
            c[2] = z
        return self.grid(c)

    def build(self):
        """(src, tgt) float32 [N,3] and the init; sources and targets are padded to the same count with far fillers at lattice
        cube centres (at least 8 u from any lattice point)."""
        src, tgt = list(self.src), list(self.tgt)
        centre = self.o + self.spacing * 0.5
        fill = 0
        while len(src) != len(tgt):
            q = centre + self.spacing * np.array([fill % 3, (fill // 3) % 3, fill // 9])
            (src if len(src) < len(tgt) else tgt).append(q - (self.delta if len(src) < len(tgt) else 0.0))
            fill += 1
        init = np.eye(4, dtype=np.float32)
        init[:3, 3] = self.delta
        return np.array(src, np.float32), np.array(tgt, np.float32), init


def radius_scene(r, origin=(0.0, 0.0, 0.0)):
    """Threshold, tie and grid edges at radius r."""
    sc = Scene(r, origin)
    u, h = sc.u, sc.h
    off = _exact_offset(sc.r2f)
    # threshold: a target at d^2 == float32(r^2) exactly is rejected ...
    c = sc.next_unit()
    j, t = sc.add(c, [c + off])
    sc.edges.append(("at r2f: rejected", j, t, False))
    # ... and one float32 step closer along the offset's main axis is kept
    c = sc.next_unit()
    q = (c + off).astype(np.float32)
    q[0] = np.nextafter(q[0], np.float32(c[0]))
    j, t = sc.add(c, [q.astype(np.float64)])
    sc.edges.append(("one float32 step inside r2f: kept", j, t, True))
    # ties: two distinct targets at exactly equal d^2 along y; the lower row sits at +a, in the cell the search visits later
    lo_y = sc.o[1]                      # the lattice's corner is the minimum on every axis
    k = np.ceil((15.0 * u) / h)
    c = sc.next_unit(y=lo_y + k * h)    # on a y cell boundary (to the grid): c - a and c + a in different cells
    a = u / 2
    j, t = sc.add(c, [c + [0, a, 0], c - [0, a, 0]])
    assert _cell(c[1] + a, lo_y, h) == _cell(c[1] - a, lo_y, h) + 1
    sc.edges.append(("tie across cells: lower row", j, t, True))
    c = sc.next_unit(y=lo_y + (k + 0.5) * h)
    a = u / 4
    j, t = sc.add(c, [c + [0, a, 0], c - [0, a, 0]])
    assert _cell(c[1] + a, lo_y, h) == _cell(c[1] - a, lo_y, h)
    sc.edges.append(("tie in one cell: lower row", j, t, True))
    # grid: sources in cell -1 of each axis, next to the lattice's corner target (the set's minimum) ...
    for ax in range(3):
        e = np.zeros(3)
        e[ax] = u / 2
        j, _ = sc.add(sc.o - e, [])
        sc.edges.append((f"cell -1 along axis {ax}", j, 0, True))
    # ... and one cell past the last one of each axis, next to a target that is that axis's maximum, high in its cell (x last:
    # every unit slot lies further along x than the ones before it)
    for ax in (1, 2, 0):
        c = sc.next_unit()
        top = max([q[ax] for q in sc.tgt] + [c[ax]]) + 4 * u
        c[ax] = sc.grid(sc.o[ax] + (np.floor((top - sc.o[ax]) / h) + 0.8) * h)
        e = np.zeros(3)
        e[ax] = u / 2
        j, t = sc.add(c + e, [c])
        sc.edges.append((f"past the last cell along axis {ax}", j, t, True))
        sc.last = getattr(sc, "last", []) + [(ax, j, t)]
    return sc


def two_cell_scene():
    """r = 0.3: float32(r^2) > r^2, so the cell side is sqrt(float32(r^2)) > r.  A kept target at a distance d between r and
    sqrt(float32(r^2)), two r-cells (but one cell) away from its source along x.  d is within 6e-9 of r: the target sits
    just above a cell boundary of side r, its source just below the one before, near x = 0 where float32 is fine enough to
    place it; the set's minimum lo (~ -0.3 k) is chosen so that the boundaries fall there."""
    r = 0.3
    sc = Scene(r)
    r2f, u = sc.r2f, sc.u
    for k in range(1, 200):                 # lo ~ -0.3 k, its boundaries lo + 0.3 k ~ 0 and lo + 0.3 (k + 1) ~ 0.3
        lo64 = np.float64(np.float32(-0.3 * k))
        q = np.float32(lo64 + 0.3 * (k + 1))
        for _ in range(4):
            q64 = np.float64(q)
            # the source: float32 just below the boundary lo + r, d^2 at least 1.5e-9 inside r2f
            p = np.float32(q64 - np.sqrt(r2f - 1.5e-9))
            while np.float64(p) > q64 - np.sqrt(r2f - 1.5e-9):
                p = np.nextafter(p, np.float32(-1.0))
            p = np.nextafter(p, np.float32(1.0))
            d = q64 - np.float64(p)
            if r < d and d * d < r2f - 1.5e-9 and _cell(q, lo64, r) - _cell(p, lo64, r) == 2:
                j, t = sc.add([np.float64(p), -3.0, -3.0], [[q64, -3.0, -3.0]])
                sc.add(np.array([lo64, -6.0, -6.0]) + sc.delta, [[lo64, -6.0, -6.0]])       # the minimum, with its own source
                sc.edges.append(("two r-cells away, kept", j, t, True))
                return sc
            q = np.nextafter(q, np.float32(1.0))
    raise AssertionError("no pair")


def status_scene(ax, cells):
    """r = 0.125 (h = 0.125): targets spanning `cells` cells along axis ax, each far target with its source next to it."""
    sc = Scene(0.125)
    far = np.zeros(3)
    far[ax] = cells * sc.h
    sc.add(far, [far])
    corner = np.full(3, (2 ** 21 - 1) * sc.h) if cells == 2 ** 21 - 1 else None
    if corner is not None:                   # all 21 key bits set on every axis
        sc.add(corner + sc.delta, [corner])
    return sc


def _oracle(src, tgt, init, r, cap, decide=None):
    return O.icp(src, tgt, init, max_correspondence_distance=r, max_iteration=cap, decide=decide, record=True)


def _first(src, tgt, init, r):
    """The oracle's first-search (row, keep) of every source."""
    seen = {}

    def decide(step, row, d2, keep):
        if step == 0:
            seen["row"], seen["keep"] = row.copy(), keep.copy()
        return row, keep
    _oracle(src, tgt, init, r, 1, decide)
    return seen["row"], seen["keep"]


def _flip(edge, tie_other):
    name, j, t, keep = edge

    def decide(step, row, d2, k):
        if step == 0:
            if tie_other is None:
                k[j] = not k[j]
            else:
                row[j] = tie_other
        return row, k
    return decide


def check_edges(sc):
    """(a) and (b) for every edge of a scene; returns the scene's arrays."""
    src, tgt, init = sc.build()
    row, keep = _first(src, tgt, init, sc.r)
    ref = _oracle(src, tgt, init, sc.r, 1)
    for e in sc.edges:
        name, j, t, want_keep = e
        assert row[j] == t and keep[j] == want_keep, (name, int(row[j]), t, bool(keep[j]))
        other = t + 1 if name.startswith("tie") else None
        flipped = _oracle(src, tgt, init, sc.r, 1, _flip(e, other))
        moved = _ulps(flipped["trans"], ref["trans"]).max()
        assert moved > FLIP_ULPS or flipped["fitness"] != ref["fitness"], (name, int(moved))
    for cap in CAPS:
        res = _oracle(src, tgt, init, sc.r, cap)
        assert res["status"] == 0 and min(res["late_margins"].values()) > MARGIN, (cap, res["late_margins"])
    return src, tgt, init


# ---------------------------------------------------------------------------------------------------
# CPU: the constructions do what they are built for
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", RADII)
def test_radius_scene_construction(r):
    sc = radius_scene(r)
    r2 = r * r
    if r == 0.10:
        assert sc.r2f < r2 and sc.h == r
    if r == 0.3:
        assert sc.r2f > r2 and sc.h == np.sqrt(sc.r2f) > r
    if r in (0.125, 1.0):
        assert sc.r2f == r2 and sc.h == r
    check_edges(sc)
    src, tgt, init = sc.build()
    lo = tgt.astype(np.float64).min(0)
    for ax, j, t in sc.last:
        p0 = src[j].astype(np.float64) + sc.delta
        assert _cell(p0[ax], lo[ax], sc.h) == _cell(tgt[:, ax], lo[ax], sc.h).max() + 1
    for name, j, _, _ in sc.edges:
        if name.startswith("cell -1"):
            ax = int(name[-1])
            assert _cell(src[j, ax] + sc.delta[ax], lo[ax], sc.h) == -1


def test_far_radius_scene_construction():
    sc = radius_scene(0.125, origin=(-10000.0, 10000.0, -10000.0))
    check_edges(sc)


def test_two_cell_scene_construction():
    sc = two_cell_scene()
    (_, j, t, _), = sc.edges
    src, tgt, init = check_edges(sc)
    p0, q = src[j].astype(np.float64) + sc.delta, tgt[t].astype(np.float64)
    d = np.linalg.norm(q - p0)
    assert sc.r < d < np.sqrt(sc.r2f)
    lo = tgt.astype(np.float64).min(0)[0]
    assert _cell(q[0], lo, sc.r) - _cell(p0[0], lo, sc.r) == 2                    # two cells of side r ...
    assert _cell(q[0], lo, sc.h) - _cell(p0[0], lo, sc.h) == 1                    # ... one of the kernel's side


@pytest.mark.parametrize("ax", [0, 1, 2])
def test_status_scene_construction(ax):
    for cells, status in ((2 ** 21 - 1, 0), (2 ** 21, 1)):
        src, tgt, init = status_scene(ax, cells).build()
        res = O.icp(src, tgt, init, max_correspondence_distance=0.125)
        assert res["status"] == status
        cc = _cell(tgt, tgt.astype(np.float64).min(0), 0.125)
        assert cc[:, ax].max() == cells
        if status == 0:
            assert (cc.max(0) == 2 ** 21 - 1).all() and min(res["margins"].values()) > MARGIN


# ---------------------------------------------------------------------------------------------------
# the other scenes, with every decision clear of its threshold (test_gpu_icp's margin gate)
# ---------------------------------------------------------------------------------------------------
def one_cell_scene():
    """r = 1: 2028 targets on a 1/16 lattice inside one cell (the N^2 path), sources next to them."""
    g = np.arange(13) / 16.0
    q = np.stack(np.meshgrid(g, g, g[:12], indexing="ij"), -1).reshape(-1, 3)
    delta = np.array([0.0, 1 / 128, 1 / 256])
    init = np.eye(4, dtype=np.float32)
    init[:3, 3] = delta
    return q.astype(np.float32), q.astype(np.float32), init, 1.0


def _mix(x):
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xff51afd7ed558ccd)
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xc4ceb9fe1a85ec53)
        x ^= x >> np.uint64(33)
    return x


def probe_chain_scene(n=512):
    """r = 0.125: n targets in distinct cells (two apart), chosen so that their keys hash (icp.cu's cell_mix, the same
    finaliser) into the first 24 of the set's 2^ceil(log2(2 n)) slots: every insertion and every lookup of an absent
    neighbour cell walks a long probe chain, wrapping around the region's end."""
    h = 0.125
    slots = 2
    while slots < 2 * n:
        slots *= 2
    i = np.arange(64)
    c = np.stack(np.meshgrid(i, i, i, indexing="ij"), -1).reshape(-1, 3).astype(np.uint64) * np.uint64(2)
    key = (c[:, 0] << np.uint64(42)) | (c[:, 1] << np.uint64(21)) | c[:, 2]
    slot = _mix(key) & np.uint64(slots - 1)
    pick = np.flatnonzero(slot < 24)
    assert len(pick) >= n
    cells = np.concatenate([[0], pick[pick != 0][:n - 1]])                  # the origin cell: lo = 0 on every axis
    q = (c[cells].astype(np.float64) + 0.5) * h
    q -= 0.5 * h                                                            # cell c's lower corner: lo + c h exactly
    q[1:] += 0.5 * h                                                        # the rest at their cells' centres
    init = np.eye(4, dtype=np.float32)
    init[:3, 3] = [0.0, 1 / 32, 1 / 64]
    return q.astype(np.float32), q.astype(np.float32), init, h, slots


def test_one_cell_and_probe_chain_constructions():
    src, tgt, init, r = one_cell_scene()
    assert len(src) == 2028 and (_cell(tgt, 0.0, O.cell_side(r)) == 0).all()
    assert O.margin(O.icp(src, tgt, init, max_correspondence_distance=r)) > MARGIN
    src, tgt, init, h, slots = probe_chain_scene()
    assert len(np.unique(_cell(tgt, 0.0, h), axis=0)) == len(tgt)
    assert O.margin(O.icp(src, tgt, init, max_correspondence_distance=h)) > MARGIN


# ---------------------------------------------------------------------------------------------------
# degenerate updates
# ---------------------------------------------------------------------------------------------------
def line_scene(kind, eps=0.0, n=16):
    """r = 0.1.  kind 'one': one correspondence (H = 0), the other sources far.  'two', 'line': n correspondences on the x
    axis, targets shifted along it by dyadic amounts.  'plane': an 8 x 8 lattice in z = const (rank-2 H).  'near_line':
    the line's sources offset along z by eps of the spread (any_perpendicular of u1 = x is y), each target a dyadic
    residual away, so that sigma_2 / sigma_1 ~ 1e-13 (test_near_line_construction)."""
    u = 1 / 16
    rng = np.random.default_rng(5)
    delta = np.array([0.0, u / 2, 0.0])
    if kind == "plane":
        g = np.arange(8) * 8 * u
        q = np.stack(np.meshgrid(g, g * 1.25, indexing="ij"), -1).reshape(-1, 2)
        tgt = np.c_[q, np.full(len(q), 0.75)]
        src = tgt - delta
    else:
        m = {"one": 1, "two": 2}.get(kind, n)
        x = np.arange(m) * 8 * u
        src = np.c_[x, np.zeros(m), np.zeros(m)]
        tgt = src + np.c_[rng.integers(-4, 5, m) / 128, np.zeros(m), np.zeros(m)]
        if kind == "one":
            src = np.r_[src, [[0.0, 0.0, 4.0], [0.0, 4.0, 0.0]]]
            tgt = np.r_[tgt, [[4.0, 0.0, 0.0], [4.0, 4.0, 4.0]]]
        if kind == "near_line":
            src[:, 2] = np.where(np.arange(m) % 3 == 0, 1.0, -0.5) * eps * 2 ** np.round(np.log2(1 + np.arange(m) % 4))
            tgt = src + delta + rng.integers(-8, 9, (m, 3)) / 256
    init = np.eye(4, dtype=np.float32)
    init[:3, 3] = delta
    return src.astype(np.float32), tgt.astype(np.float32), init, 0.1


def _near_line_eps():
    """eps that puts the first update's sigma_2 / sigma_1 near 1e-13 (sigma_2 grows linearly with eps)."""
    src, tgt, init, r = line_scene("near_line", 2.0 ** -30)
    ratio = O.icp(src, tgt, init, max_correspondence_distance=r, max_iteration=1)["margins"]["sigma_ratio"]
    return 2.0 ** np.round(np.log2(2.0 ** -30 * 1e-13 / ratio))


def test_near_line_construction():
    src, tgt, init, r = line_scene("near_line", _near_line_eps())
    res = O.icp(src, tgt, init, max_correspondence_distance=r, record=True)
    assert res["fitness"] == 1.0
    a, b = res["updates"][0]
    s = np.linalg.svd((a - a.mean(0)).T @ (b - b.mean(0)), compute_uv=False)
    assert 1e-14 <= s[1] / s[0] <= 1e-12, s
    late = res["late_margins"]
    assert min(late["d2_radius"], late["nn_gap"], late["rmse_criterion"]) > MARGIN
    _, T, tol_R, _, _, _ = near_line_reference(src, tgt, init, r)
    assert tol_R < 0.1, tol_R


# ---------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------
def _device(src, tgt, init, r, cap):
    from pointdsc_b200.icp import icp_refine_packed
    out, info = icp_refine_packed(torch.from_numpy(np.ascontiguousarray(src)).cuda(), torch.from_numpy(np.ascontiguousarray(tgt)).cuda(),
                                  torch.from_numpy(np.asarray(init, np.float32).reshape(1, 4, 4)).cuda(), [0, len(src)], info=True,
                                  max_correspondence_distance=r, max_iteration=cap)
    return (out[0].cpu().numpy(), float(info["fitness"][0]), float(info["inlier_rmse"][0]), int(info["iterations"][0]),
            int(info["status"][0]))


# test_gpu_icp._check's parity (rmse 1e-12 relative, T 2 float32 ulps) plus absolute slacks for what these sets add: tiny
# rotation entries (R ~ I here, where 2 ulps of 1e-19 say nothing) and coordinates up to 2.6e5 (the cell-limit sets).  The
# two float64 runs differ per update by <= (C_SVD + 6 C_PRE) eps64 s1 / (s2 + d s3) in R (test_gpu_kabsch's solver and
# pre-solver terms, 16 + 6 * 32 = 208), summed over the updates (`_kappa`); that moves t = cb - R ca by 3 |dR| M, M the
# largest coordinate, and the residuals by 4 |dR| M; the centroids add <= 14 eps64 M each (icp_block_sum), K_ABS = 32 covers
# them.  Measured on an H100 (80 GB HBM3, 700 W): the worst error is 0.25 of these tolerances (printed per set).
K_R, K_ABS = 208.0, 32.0


def _kappa(ref):
    """Sum over the run's updates of s1 / (s2 + d s3) of H (0 for H = 0, where both sides return R = I exactly)."""
    k = 0.0
    for a, b in ref["updates"]:
        H = (a - a.mean(0)).T @ (b - b.mean(0))
        if np.any(H):
            U, sv, Vt = np.linalg.svd(H)
            d = np.sign(np.linalg.det(Vt.T @ U.T))
            k += sv[0] / (sv[1] + d * sv[2])
    return k


def _parity(dev, ref, what, M):
    trans, fit, rmse, its, status = dev
    dR = K_R * EPS64 * _kappa(ref)
    slack = np.zeros((4, 4))
    slack[:3, :3] = dR
    slack[:3, 3] = 3.0 * dR * M + K_ABS * EPS64 * M
    slack_rmse = 4.0 * dR * M + K_ABS * EPS64 * M
    assert status == ref["status"], what
    assert its == ref["iterations"], (what, its, ref["iterations"])
    assert fit == ref["fitness"], (what, fit, ref["fitness"])
    err_rmse = abs(rmse - ref["inlier_rmse"])
    assert err_rmse <= 1e-12 * ref["inlier_rmse"] + slack_rmse, (what, rmse, ref["inlier_rmse"])
    err = np.abs(trans - ref["trans64"])
    ok = (_ulps(trans, ref["trans"]) <= 2) | (err <= slack)
    assert ok.all(), (what, trans, ref["trans"], slack)
    return max(err_rmse / (1e-12 * ref["inlier_rmse"] + slack_rmse),
               float((err / (slack + 2 * np.spacing(np.abs(ref["trans"])))).max()))


def _mag(src, tgt, init):
    return float(max(np.abs(src).max(), np.abs(tgt).max(), np.abs(init).max()))


def _run_scene(src, tgt, init, r, what):
    worst = 0.0
    for cap in CAPS:
        ref = _oracle(src, tgt, init, r, cap)
        worst = max(worst, _parity(_device(src, tgt, init, r, cap), ref, f"{what} cap={cap}", _mag(src, tgt, init)))
    print(f"{what}: worst rmse / translation error over its tolerance {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("r", RADII)
def test_radius_edges(r):
    sc = radius_scene(r)
    _run_scene(*check_edges(sc), r, f"r={r}")


@pytest.mark.gpu
def test_radius_edges_far_from_the_origin():
    sc = radius_scene(0.125, origin=(-10000.0, 10000.0, -10000.0))
    _run_scene(*check_edges(sc), 0.125, "+-1e4")


@pytest.mark.gpu
def test_kept_target_two_r_cells_away():
    sc = two_cell_scene()
    _run_scene(*check_edges(sc), sc.r, "two cells")


@pytest.mark.gpu
@pytest.mark.parametrize("ax", [0, 1, 2])
def test_cell_limit(ax):
    for cells in (2 ** 21 - 1, 2 ** 21):
        src, tgt, init = status_scene(ax, cells).build()
        for cap in CAPS:
            ref = _oracle(src, tgt, init, 0.125, cap)
            dev = _device(src, tgt, init, 0.125, cap)
            assert dev[4] == (0 if cells < 2 ** 21 else 1), (ax, cells, dev[4])
            _parity(dev, ref, f"axis {ax} cells {cells}", _mag(src, tgt, init))


@pytest.mark.gpu
def test_one_cell_and_long_probe_chains():
    src, tgt, init, r = one_cell_scene()
    _run_scene(src, tgt, init, r, "one cell")
    src, tgt, init, h, _ = probe_chain_scene()
    _run_scene(src, tgt, init, h, "probe chains")


@pytest.mark.gpu
@pytest.mark.parametrize("r", [0.3, 0.125, 1.0, 1e-3])
def test_synthetic_pairs_at_other_radii(r):
    """test_gpu_icp's pairs at the other radii, under its margin gate (every case below clears it at every radius)."""
    from pointdsc_b200.synth import make_pair
    for preset, n, seed in [("3dmatch", 41, 0), ("3dmatch", 1000, 0), ("3dmatch", 5000, 2), ("kitti", 41, 0), ("kitti", 1000, 0)]:
        p = make_pair(seed, n, preset)
        src, tgt, gt = p["src_keypts"].numpy(), p["tgt_keypts"].numpy(), p["gt_trans"].numpy().astype(np.float32)
        ref = _oracle(src, tgt, gt, r, 30)
        assert O.margin(ref) > MARGIN, (preset, n, seed, ref["margins"])
        _parity(_device(src, tgt, gt, r, 30), ref, f"{preset} n={n} r={r}", _mag(src, tgt, gt))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["one", "plane"])
def test_translation_only_and_rank2_updates(kind):
    src, tgt, init, r = line_scene(kind)
    for cap in CAPS:
        ref = _oracle(src, tgt, init, r, cap)
        assert O.margin(ref) > MARGIN, ref["margins"]
        _parity(_device(src, tgt, init, r, cap), ref, kind, _mag(src, tgt, init))
    if kind == "one":
        assert np.array_equal(_device(src, tgt, init, r, 1)[0][:3, :3], np.eye(3, dtype=np.float32))   # H = 0: R = I


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["two", "line"])
def test_collinear_updates(kind):
    """Exactly collinear correspondences: the rotation about the line is not unique, so the device and the oracle may pick
    different ones.  What is unique is checked: R is a rotation, T maps every source point (all on the line) where the
    oracle's T does, and fitness, rmse and the iterations are the oracle's.  Tolerance of the mapped points: T comes back in
    float32, each of its 12 entries rounded (2^-24 relative), so |T s - T64 s| <= 2^-24 (|R| |s|_1 + |t|) per coordinate;
    2^-22 (|s|_1 + |t|max) covers it and the float64 differences (~1e-15) with 2x to spare."""
    src, tgt, init, r = line_scene(kind)
    for cap in CAPS:
        ref = O.icp(src, tgt, init, max_correspondence_distance=r, max_iteration=cap)
        trans, fit, rmse, its, status = _device(src, tgt, init, r, cap)
        assert status == 0 and its == ref["iterations"] and fit == ref["fitness"] == 1.0
        assert abs(rmse - ref["inlier_rmse"]) <= 1e-12 * ref["inlier_rmse"]
        R = trans[:3, :3].astype(np.float64)
        assert np.abs(R @ R.T - np.eye(3)).max() <= 1e-6 and abs(np.linalg.det(R) - 1) <= 1e-6
        s = src.astype(np.float64)
        got = s @ R.T + trans[:3, 3]
        want = s @ ref["trans64"][:3, :3].T + ref["trans64"][:3, 3]
        tol = 2.0 ** -22 * (np.abs(s).sum(1) + np.abs(trans[:3, 3]).max())
        assert (np.abs(got - want).max(1) <= tol).all(), (kind, cap, np.abs(got - want).max())
        # the centroids: the moved source centroid lands on the oracle's
        assert np.abs(got.mean(0) - want.mean(0)).max() <= tol.max()


def near_line_reference(src, tgt, init, r):
    """The first update of the near-collinear set, solved in long double (test_gpu_kabsch.kabsch_ld: LAPACK's float64 SVD is
    itself off by ~50 eps64 s1 / (s2 + d s3), 0.1 here), composed with the init, and the bound of the device's T against it:
        |R - R_ref| <= C_SVD eps64 s1 / (s2 + d s3) + |Omega|_F,   Omega_ij = (E'_ij - E'_ji) / (s~_i + s~_j),
    s~ = (s1, s2, d s3), E' = |U|^T E |V| the error of the device's float64 H in H's singular frame, E its entrywise bound.
    Omega is the first-order change of the polar factor under H + E.  The device's H (icp.cu) sums the products of
    m = P - ca and n = q - cb: the centroids' errors cancel to first order (the centred points sum to N times that error, so
    they enter H as N dca dcb^T), the subtractions round relative to m and n, and the products and the fixed-order sum add
    <= 14 eps64 (one term per thread, a 5-level warp tree, 8 warps): E_ij <= C_PRE eps64 sum_k |m_ki| |n_kj|, C_PRE = 32.  E
    lies along the line (the x row), which the near-zero pair s2, s3 does not see: the bound stays far below 1."""
    from test_gpu_kabsch import C_PRE, C_SVD, kabsch_ld
    ref = O.icp(src, tgt, init, max_correspondence_distance=r, max_iteration=1, record=True)
    a, b = (x.astype(np.longdouble) for x in ref["updates"][0])
    ca, cb = a.mean(0), b.mean(0)
    m, n = a - ca, b - cb
    H = (m.T @ n).astype(np.float64)
    R, s, d, U, V = (x[0] for x in kabsch_ld(H[None]))
    t = (cb - R.astype(np.longdouble) @ ca).astype(np.float64)
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    T = T @ init.astype(np.float64)
    mf, nf = np.abs(m.astype(np.float64)), np.abs(n.astype(np.float64))
    E = C_PRE * EPS64 * (mf.T @ nf)
    Ep = np.abs(U).T @ E @ np.abs(V)
    st = np.array([s[0], s[1], d * s[2]])
    omega = sum(((Ep[i, j] + Ep[j, i]) / (st[i] + st[j])) ** 2 for i in range(3) for j in range(3) if i != j) ** 0.5
    tol_R = C_SVD * EPS64 * s[0] / (s[1] + d * s[2]) + omega
    Ma, Mb = float(np.abs(a).max()), float(np.abs(b).max())
    return ref, T, tol_R, s, Ma, Mb


@pytest.mark.gpu
def test_near_collinear_update_against_the_polar_bound():
    """sigma_2 / sigma_1 ~ 1e-13 in the first update: the double solver must take u2 from H (before its rank threshold was
    scaled to double it made u2 up, and R was off by up to 2 about the line).  One update against the long-double reference
    within `near_line_reference`'s bound, then the full run: fitness, rmse and the iterations are the oracle's (the rotation
    about the line moves no point by more than ~1e-13 of the spread, so no correspondence changes).  Measured on an H100
    (80 GB HBM3, 700 W): s2 / s1 = 1.06e-13, bound 0.034, |R - R_ref| = 4.7e-7 of it; before the fix the update missed it."""
    src, tgt, init, r = line_scene("near_line", _near_line_eps())
    ref, T, tol_R, s, Ma, Mb = near_line_reference(src, tgt, init, r)
    assert tol_R < 0.1, tol_R                                             # far from vacuous: a made-up u2 is off by ~1
    trans, fit, rmse, its, status = _device(src, tgt, init, r, 1)
    assert status == 0 and its == 1 and fit == ref["fitness"]
    err_R = np.abs(trans[:3, :3] - T[:3, :3]).max()
    tol_R32 = tol_R + 2.0 ** -23                                          # plus T's float32 rounding
    assert err_R <= tol_R32, (err_R, tol_R32, s[1] / s[0])
    # t = cb - R ca: the rotation's error at the centroid, the centroids' own (<= 14 eps64 M each) and float32 rounding
    tol_t = 3.0 * tol_R * Ma + 32.0 * EPS64 * (Ma + Mb) + 2.0 ** -23 * np.abs(T[:3, 3]).max()
    err_t = np.abs(trans[:3, 3] - T[:3, 3]).max()
    assert err_t <= tol_t, (err_t, tol_t)
    print(f"near-collinear: s2/s1 = {s[1] / s[0]:.3g}, bound {tol_R:.3g}, |R - R_ref| / bound = {err_R / tol_R32:.3g}, "
          f"|t - t_ref| / bound = {err_t / tol_t:.3g}")
    full = O.icp(src, tgt, init, max_correspondence_distance=r)
    trans, fit, rmse, its, status = _device(src, tgt, init, r, 30)
    assert status == 0 and its == full["iterations"] and fit == full["fitness"]
    assert abs(rmse - full["inlier_rmse"]) <= 1e-12 * full["inlier_rmse"] + K_ABS * EPS64 * _mag(src, tgt, init)
