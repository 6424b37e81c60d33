"""Helpers shared by the CPU and GPU tests of the marker-triplet drone locator (csrc/locate_device.cuh,
csrc/locate_kernels.cu) and the golden generator tests/golden/make_golden_locate.py: seeded scenes that reach every
branch of the greedy scan (crowded rigs, shared markers, tolerance edges ulp by ulp, heading folds, the drone-index
edge, count limits, non-finite rows, random fuzz), the oracle on a scene as arrays, a trace of which points the scan
picked (for the reach statistics) and the comparison both test tiers use.

A scene is (points f64 [K, 3], errors f64 [K]); a batch is (obj f64 [B, R, 3], err f64 [B, R], n int32 [B]) in the
layout mocap_locate_objects_dev reads, its rows beyond n filled with a marker triplet that must be ignored."""
import os

import numpy as np

from oracle.ref_port import RefPort
from tests.hostbuild import ptr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "locate_edge.npz")
D1, D2, TOL = 0.095, 0.15, 0.025
HALF = D2 / 2
APEX = float(np.sqrt(D1 ** 2 - HALF ** 2))      # distance of the third marker from the pair's axis
ULP_HALF_PI = float(np.spacing(np.pi / 2))
HEADING_TOL = 4 * ULP_HALF_PI                   # atan2 of the device / glibc / numpy: a few ulps of pi / 2 at most
SCAN = 8                                        # ulps either side of a tolerance edge
MAX_POINTS = 128                                # MOCAP_MAX_ROOTS
FUZZ_SCENES = 2000
GOLDEN_FUZZ = 300


# ---------------------------------------------------------------------------------------------- pieces
def _errors(rng, k):
    return rng.uniform(0.05, 2.0, k)


def _rotation(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    return q


def triplet(centre, R=None, side=1.0):
    """Rows a, b (0.15 apart along the local x axis) and the apex, 0.095 from both."""
    local = np.array([[HALF, 0, 0], [-HALF, 0, 0], [0, side * APEX, 0]])
    return local @ (np.eye(3) if R is None else R).T + np.asarray(centre, dtype=np.float64)


def _stepped(x, k):
    """x moved by k ulps."""
    for _ in range(abs(k)):
        x = np.nextafter(x, np.inf if k > 0 else -np.inf)
    return float(x)


def _scene(rows, seed):
    pts = np.ascontiguousarray(np.asarray(rows, dtype=np.float64).reshape(-1, 3))
    return pts, _errors(np.random.default_rng(seed), len(pts))


# ---------------------------------------------------------------------------------------------- crowded rigs
def crowded(n_drones, box, seed, n_clutter=0, K=None, jitter=0.004, place=None, near=0.5):
    """n_drones triplets at random attitudes in a box of side `box` (small: markers of different drones fall 0.095 +-
    0.025 apart, so points have three and more neighbours and triplets share markers), each new drone beside an earlier
    one with probability `near`; clutter; shuffled; cut or filled with clutter to K points.  place = (i, a, b): drone
    0, set apart from the crowd so that the scan finds it as such, has its apex and pair moved to these rows."""
    rng = np.random.default_rng(seed)
    pts, centres = [], []
    for d in range(n_drones):
        if centres and rng.uniform() < near:
            off = rng.normal(size=3)
            c = centres[rng.integers(len(centres))] + off / np.linalg.norm(off) * rng.uniform(0.06, 0.2)
        else:
            c = rng.uniform(-box / 2, box / 2, 3)
        if place is not None and d == 0:
            c = c + [2.0, 0.0, 0.0]
        else:
            centres.append(c)
        pts.extend(triplet(c, _rotation(rng), rng.choice([-1.0, 1.0])) + rng.uniform(-jitter, jitter, (3, 3)))
    pts.extend(rng.uniform(-box / 2, box / 2, (n_clutter, 3)))
    pts = np.array(pts, dtype=np.float64).reshape(-1, 3)
    drone0 = pts[:3].copy()
    pts = pts[rng.permutation(len(pts))][:K]
    if K is not None and len(pts) < K:
        pts = np.vstack([pts, rng.uniform(-box / 2, box / 2, (K - len(pts), 3))])
    if place is not None:
        for row, dst in zip(drone0[[2, 0, 1]], place):              # apex, a, b
            cur = int(np.flatnonzero((pts == row).all(axis=1))[0])
            pts[[cur, dst]] = pts[[dst, cur]]
    return np.ascontiguousarray(pts), _errors(rng, len(pts))


# ---------------------------------------------------------------------------------------------- shared markers
def chain(n, seed=0):
    """A zigzag: consecutive points 0.095 apart, every other one 0.15 apart.  Every odd point becomes an object whose
    pair is its two neighbours, so consecutive objects share a marker that is already on the matched list."""
    return _scene([[k * HALF, (k % 2) * APEX, 0.3] for k in range(n)], seed)


def fan(seed=0, order=None):
    """A hub and a ring of 7 points 0.095 around it: ring neighbours are 0.082 apart (inside the neighbour tolerance),
    next-but-one 0.149 apart (a pair), so the hub has 7 neighbours and every ring point 3.  `order` permutes the rows."""
    ang = 2 * np.pi * np.arange(7) / 7
    rows = np.vstack([[0.0, 0.0, 0.0], np.stack([D1 * np.cos(ang), D1 * np.sin(ang), np.zeros(7)], axis=1)]) + [0.2, -0.1, 0.4]
    pts, errs = _scene(rows, seed)
    if order is not None:
        pts = np.ascontiguousarray(pts[list(order)])
    return pts, errs


def lattice(rows, cols, seed=0):
    """Isosceles tiles (base 0.15, legs 0.095), rows offset by half a base, indexed row by row: a point's first pair in
    index order lies in the row above, which the scan has already passed, so nearly every point becomes an object --
    the reference's one-object-per-point ceiling."""
    return _scene([[c * D2 + (r % 2) * HALF, -r * APEX, 0.1] for r in range(rows) for c in range(cols)], seed)


# ---------------------------------------------------------------------------------------------- tolerance edges
def neighbour_scan(edge):
    """Point 0 at the origin, point 1 on the x axis at `edge` (0.070 or 0.120: the ends of the neighbour test) moved
    -SCAN .. SCAN ulps, point 2 placed 0.095 from point 0 and 0.15 from point 1.  One object exactly when point 1 passes
    the neighbour test.  Returns the 2 * SCAN + 1 scenes."""
    x = (edge ** 2 + D1 ** 2 - D2 ** 2) / (2 * edge)
    third = [x, float(np.sqrt(D1 ** 2 - x ** 2)), 0.0]
    return [_scene([[0.0, 0.0, 0.0], [_stepped(edge, k), 0.0, 0.0], third], 1000 + k) for k in range(-SCAN, SCAN + 1)]


def pair_scan(edge):
    """Point 1 at the origin, point 2 on the x axis at `edge` (0.125 or 0.175: the ends of the pair test) moved -SCAN ..
    SCAN ulps, point 0 the apex 0.095 from both.  One object exactly when the pair is not refused."""
    apex = [edge / 2, float(np.sqrt(D1 ** 2 - (edge / 2) ** 2)), 0.0]
    return [_scene([apex, [0.0, 0.0, 0.0], [_stepped(edge, k), 0.0, 0.0]], 2000 + k) for k in range(-SCAN, SCAN + 1)]


def tolerance_scenes():
    """name -> scene for the four scans.  Asserts that the oracle's decision flips inside each scan: the scan straddles
    the edge in floating point."""
    out = {}
    for kind, build, edges in (("neighbour", neighbour_scan, (0.070, 0.120)), ("pair", pair_scan, (0.125, 0.175))):
        for edge in edges:
            scenes = build(edge)
            counts = [oracle(*sc)[0] for sc in scenes]
            assert set(counts) == {0, 1} and counts[0] != counts[-1], (kind, edge, counts)
            assert sum(counts[i] != counts[i + 1] for i in range(2 * SCAN)) == 1, (kind, edge, counts)
            for k, sc in zip(range(-SCAN, SCAN + 1), scenes):
                out[f"{kind}_{edge:.3f}_{k:+d}ulp"] = sc
    return out


# ---------------------------------------------------------------------------------------------- heading, drone index
def _pair_scene(a, b, apex, swap, seed):
    """Rows apex, a, b (or apex, b, a): the scan takes the pair in row order, so both signs of a - b occur."""
    return _scene([apex, b, a] if swap else [apex, a, b], seed)


def heading_scenes():
    """name -> scene.  Pairs along +-y exactly (atan2 gives +-pi/2, which the strict folds keep), 1 .. 3 ulps of
    heading either side of +-y (names starting "heading_near_y": the fold may or may not apply there), along +-x and
    vertical (atan2(0, 0)); both marker orders of each."""
    out = {}
    c = np.array([0.4, -0.2, 0.7])
    for swap in (False, True):
        tag = "ba" if swap else "ab"
        out[f"heading_y_{tag}"] = _pair_scene(c + [0, HALF, 0], c + [0, -HALF, 0], c + [APEX, 0, 0], swap, 31)
        out[f"heading_x_{tag}"] = _pair_scene(c + [HALF, 0, 0], c + [-HALF, 0, 0], c + [0, APEX, 0], swap, 32)
        out[f"heading_vertical_{tag}"] = _pair_scene(c + [0, 0, HALF], c + [0, 0, -HALF], c + [APEX, 0, 0], swap, 33)
        for k in (-3, -2, -1, 1, 2, 3):
            # a - b = (k ulps of pi/2 times 0.15, 0.15, 0): the heading lies k ulps from the fold; around the origin, so
            # that the tiny x offset is not rounded away
            dx = k * D2 * ULP_HALF_PI
            out[f"heading_near_y_{k:+d}_{tag}"] = _pair_scene([dx, HALF, 0], [0.0, -HALF, 0], [APEX, 0, 0], swap, 40 + k)
    return out


def index_scenes():
    """The apex at exactly the pair's mean y (droneIndex 1: the test is a strict >) and one ulp either side."""
    out = {}
    y = 0.3
    for k in (-1, 0, 1):
        out[f"index_{k:+d}ulp"] = _scene([[0.0, _stepped(y, k), APEX], [HALF, y, 0.0], [-HALF, y, 0.0]], 50 + k)
    return out


# ---------------------------------------------------------------------------------------------- non-finite rows
def nonfinite_scenes():
    """Two drones and clutter with a NaN row, an inf row, or both, at rows the scan meets before, between and after
    the drones' markers."""
    out = {}
    for name, bad in (("nan", [[np.nan, 0.1, 0.2]]), ("inf", [[0.1, -np.inf, 0.2]]),
                      ("nan_inf", [[np.nan, np.nan, np.nan], [np.inf, np.inf, 0.0], [0.0, 0.0, -np.inf]])):
        for at in (0, 4, None):
            pts, errs = crowded(2, 0.25, seed=61, n_clutter=3, near=1.0)
            rows = np.asarray(bad, dtype=np.float64)
            k = len(pts) if at is None else at
            pts = np.ascontiguousarray(np.vstack([pts[:k], rows, pts[k:]]))
            errs = np.concatenate([errs[:k], np.full(len(rows), 0.5), errs[k:]])
            out[f"nonfinite_{name}_at_{'end' if at is None else at}"] = (pts, errs)
    return out


# ---------------------------------------------------------------------------------------------- the named scenes
_cache = {}


def small_scenes():
    """The deterministic scenes of at most 16 points: shared markers, tolerance edges, heading, drone index,
    non-finite rows, and frame-sets of 0, 1 and 2 points."""
    if "small" not in _cache:
        s = {"empty": (np.zeros((0, 3)), np.zeros(0)), "one_point": _scene([[0.1, 0.2, 0.3]], 70),
             "two_points": _scene([[0.0, 0.0, 0.0], [D1, 0.0, 0.0]], 71),
             "chain_16": chain(16), "fan": fan(), "fan_hub_last": fan(order=[3, 1, 6, 2, 7, 5, 4, 0]),
             "fan_hub_mid": fan(order=[5, 2, 7, 0, 1, 6, 3, 4]), "lattice_4x4": lattice(4, 4)}
        s.update(tolerance_scenes())
        s.update(heading_scenes())
        s.update(index_scenes())
        s.update(nonfinite_scenes())
        assert all(len(p) <= 16 for p, _ in s.values())
        _cache["small"] = s
    return _cache["small"]


def large_scenes():
    """The deterministic scenes of up to 128 points: crowded rigs (three of them with drone 0's apex and pair moved to
    rows that straddle 63 / 64 and use 127), a long chain and the lattices."""
    if "large" not in _cache:
        s = {"crowded_20": crowded(20, 0.45, seed=81, n_clutter=10),
             "crowded_30": crowded(30, 0.5, seed=82, n_clutter=20, K=100),
             "crowded_40_full": crowded(40, 0.55, seed=83, n_clutter=30, K=MAX_POINTS),
             "crowded_jitter": crowded(36, 0.5, seed=84, n_clutter=20, K=MAX_POINTS, jitter=0.02),
             "straddle_63_64_127": crowded(40, 0.6, seed=85, n_clutter=8, K=MAX_POINTS, place=(63, 64, 127)),
             "straddle_127_62_65": crowded(40, 0.6, seed=86, n_clutter=8, K=MAX_POINTS, place=(127, 62, 65)),
             "straddle_64_0_127": crowded(38, 0.6, seed=87, n_clutter=14, K=MAX_POINTS, place=(64, 0, 127)),
             "chain_128": chain(MAX_POINTS, seed=3), "lattice_8x16": lattice(8, 16, seed=4),
             "lattice_16x8": lattice(16, 8, seed=5), "lattice_5x13": lattice(5, 13, seed=6)}
        for name, place in (("straddle_63_64_127", (63, 64, 127)), ("straddle_127_62_65", (127, 62, 65)),
                            ("straddle_64_0_127", (64, 0, 127))):
            assert place in [t for t in trace(s[name][0])["triplets"]], name      # that very triplet is found
        for name in ("lattice_8x16", "lattice_16x8", "lattice_5x13"):
            assert oracle(*s[name])[0] >= 0.7 * len(s[name][0]), name
        _cache["large"] = s
    return _cache["large"]


def edge_scenes():
    """Every named scene, small ones first."""
    return {**small_scenes(), **large_scenes()}


def fuzz_scenes(count=FUZZ_SCENES, seed=2026):
    """0-40 drones (each new one beside an earlier one with probability one half) and 0-30 clutter points in a box sized
    to the drone count, jitter up to 0.02, cut to 128 points."""
    key = ("fuzz", count, seed)
    if key not in _cache:
        rng = np.random.default_rng(seed)
        out = []
        for s in range(count):
            nd, nc = int(rng.integers(0, 41)), int(rng.integers(0, 31))
            box = float(rng.uniform(0.3, 1.2))
            K = min(MAX_POINTS, 3 * nd + nc)
            out.append(crowded(nd, box, seed=seed * 10000 + s, n_clutter=nc, K=K, jitter=float(rng.uniform(0, 0.02))))
        _cache[key] = out
    return _cache[key]


def golden_fuzz_scenes():
    """The sample of the fuzz the real reference was run on: every 6th scene, GOLDEN_FUZZ of them."""
    return fuzz_scenes()[::6][:GOLDEN_FUZZ]


# ---------------------------------------------------------------------------------------------- batches
DECOY = triplet([0.0, 0.0, 0.0])[[2, 0, 1]]        # apex, a, b: an object if a scan ever reads it


def pack(scenes, R, n=None):
    """Scenes -> (obj [B, R, 3], err [B, R], n [B]); the rows beyond a scene's points hold the decoy triplet over and
    over.  n overrides the counts (None entries keep the scene's)."""
    B = len(scenes)
    obj = np.empty((B, R, 3)); err = np.full((B, R), 0.25); cnt = np.zeros(B, np.int32)
    obj[:] = DECOY[np.arange(R) % 3]
    for s, (p, e) in enumerate(scenes):
        k = len(p)
        assert k <= R, (k, R)
        obj[s, :k] = p; err[s, :k] = e
        cnt[s] = k if n is None or n[s] is None else n[s]
    return obj, err, cnt


def count_cases(R):
    """(scenes as the locator must see them, batch) for frame-set counts 0, 1, 2, R, R + 5 and -1 over rows that hold
    valid triplets throughout.  The R + 5 frame-set is followed by one that starts with a triplet: reading past R
    rows would find it."""
    full = crowded(R // 3, 0.5, seed=91, n_clutter=R // 8 + 1, K=R)
    over = (np.ascontiguousarray(np.vstack([triplet([0.3, 0.3, 0.3]), np.tile([[5.0, 5.0, 5.0]], (R - 3, 1))
                                            + np.arange(R - 3)[:, None] * [1.0, 0.0, 0.0]])), np.linspace(0.1, 1.0, R))
    after = _scene(np.vstack([triplet([9.0, 9.0, 9.0]), [[0.0, 7.0, 0.0]]]), 92)
    rows = [(full, 0), (full, 1), (full, 2), (full, R), (over, R + 5), (after, None), (full, -1), (chain(min(R, 12)), None)]
    obj, err, n = pack([sc for sc, _ in rows], R, [k for _, k in rows])
    seen = []
    for (p, e), k in rows:
        k = len(p) if k is None else max(0, min(k, R))
        seen.append((p[:k], e[:k]))
    return seen, (obj, err, n)


# ---------------------------------------------------------------------------------------------- oracle
def oracle(pts, errs, max_objects=None):
    """RefPort.locate_objects on one scene as (count, records f64 [count, 5] = x y z heading error, drone_index int32
    [count]), cut to the first max_objects."""
    key = (pts.tobytes(), errs.tobytes())
    if key not in _cache:
        with np.errstate(invalid="ignore"):
            found = RefPort.locate_objects(pts.copy(), errs.copy()) if len(pts) else []
        rec = np.zeros((len(found), 5)); di = np.zeros(len(found), np.int32)
        for i, o in enumerate(found):
            rec[i, :3], rec[i, 3], rec[i, 4], di[i] = o["pos"], o["heading"], o["error"], o["droneIndex"]
        _cache[key] = (rec, di)
    rec, di = _cache[key]
    k = len(rec) if max_objects is None else min(len(rec), max_objects)
    return k, rec[:k], di[:k]


def trace(pts):
    """Which rows the greedy scan picks, for the reach statistics only (the tests compare against `oracle`):
    triplets [(i, a, b)], shared = objects whose a or b was already on the matched list, many = points with three or
    more neighbours, high = objects with a row >= 64 among i, a, b, screened_high = rows >= 64 skipped as i."""
    K = len(pts)
    with np.errstate(invalid="ignore"):
        dist = np.sqrt(((pts[:, None, :] - pts[None, :, :]) ** 2).sum(axis=2)) if K else np.zeros((0, 0))
        near = np.abs(dist - D1) < TOL
        pair_ok = ~(np.abs(dist - D2) > TOL)
    used, out = set(), dict(triplets=[], shared=0, many=int((near.sum(axis=1) >= 3).sum()), high=0, screened_high=0)
    for i in range(K):
        if i in used:
            out["screened_high"] += i >= 64
            continue
        m = np.flatnonzero(near[i])
        if len(m) < 2:
            continue
        ok = pair_ok[np.ix_(m, m)]
        if not ok.any():
            continue
        ia, ib = np.unravel_index(int(np.argmax(ok)), ok.shape)       # first True in row-major order
        a, b = int(m[ia]), int(m[ib])
        out["shared"] += (a in used) or (b in used)
        out["high"] += max(i, a, b) >= 64
        used.update((i, a, b))
        out["triplets"].append((i, a, b))
    return out


SENTINEL_F, SENTINEL_I = -7.25e300, -123456789
GUARD = 3                                          # sentinel rows after every frame-set's records


def guarded_outputs(B, max_objects, xp=np, **kw):
    """Outputs with GUARD sentinel rows after every frame-set's records, and behind the last frame-set as many more
    sentinel slabs as the longest possible overrun (one object per point) would cross, so that a missing bound shows
    as a changed sentinel rather than a fault: rec [B + T, max_objects + GUARD, 5], di [B + T, max_objects + GUARD],
    n [B + GUARD], filled with sentinels.  xp is numpy or torch."""
    T = -(-MAX_POINTS // (max_objects + GUARD))
    rec = xp.full((B + T, max_objects + GUARD, 5), SENTINEL_F, dtype=xp.float64, **kw)
    di = xp.full((B + T, max_objects + GUARD), SENTINEL_I, dtype=xp.int32, **kw)
    n = xp.full((B + GUARD,), SENTINEL_I, dtype=xp.int32, **kw)
    return rec, di, n


def host_locate(lib, obj, err, n, max_roots, max_objects):
    """The host build on a batch, one frame-set per call into its own guarded slab: dict objects [B, max_objects, 5],
    drone_index [B, max_objects], n [B].  Asserts that every guard row and every record slot at or beyond n is
    untouched."""
    obj = np.ascontiguousarray(obj, np.float64); err = np.ascontiguousarray(err, np.float64); n = np.ascontiguousarray(n, np.int32)
    B = len(n)
    rec, di, cnt = guarded_outputs(B, max_objects)
    # frame-set s writes rec[s, :max_objects]: the library sees a batch of one whose outputs start at that row
    for s in range(B):
        lib.hc_locate(ptr(obj[s:]), ptr(err[s:]), ptr(n[s:]), 1, max_roots, max_objects, ptr(rec[s:]), ptr(di[s:]), ptr(cnt[s:]))
    check_guards(rec, di, cnt, B, max_objects)
    return {"objects": rec[:B, :max_objects].copy(), "drone_index": di[:B, :max_objects].copy(), "n": cnt[:B].copy()}


def host_locate_batch(lib, obj, err, n, max_roots, max_objects):
    """The host build on a whole batch in one call, outputs in the dense layout of mocap_locate_objects_dev followed by
    one guard slab."""
    obj = np.ascontiguousarray(obj, np.float64); err = np.ascontiguousarray(err, np.float64); n = np.ascontiguousarray(n, np.int32)
    B = len(n)
    rec = np.full((B + 1, max_objects, 5), SENTINEL_F); di = np.full((B + 1, max_objects), SENTINEL_I, np.int32)
    cnt = np.full(B + 1, SENTINEL_I, np.int32)
    lib.hc_locate(ptr(obj), ptr(err), ptr(n), B, max_roots, max_objects, ptr(rec), ptr(di), ptr(cnt))
    assert (rec[B] == SENTINEL_F).all() and (di[B] == SENTINEL_I).all() and cnt[B] == SENTINEL_I
    return {"objects": rec[:B], "drone_index": di[:B], "n": cnt[:B]}


def check_guards(rec, di, cnt, B, max_objects):
    """numpy arrays of guarded_outputs after a run: guard rows, the slabs behind the last frame-set, the count's tail
    and the record slots at or beyond each frame-set's count still hold the sentinels."""
    assert (rec[:B, max_objects:] == SENTINEL_F).all() and (di[:B, max_objects:] == SENTINEL_I).all()
    assert (rec[B:] == SENTINEL_F).all() and (di[B:] == SENTINEL_I).all() and (cnt[B:] == SENTINEL_I).all()
    assert ((cnt[:B] >= 0) & (cnt[:B] <= max_objects)).all()
    beyond = np.arange(max_objects)[None, :] >= cnt[:B, None]
    assert (rec[:B, :max_objects][beyond] == SENTINEL_F).all() and (di[:B, :max_objects][beyond] == SENTINEL_I).all()


# ---------------------------------------------------------------------------------------------- comparison
def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def fold_allowed(name):
    """The only scenes whose heading may differ from the oracle's by pi: the pair lies 1 .. 3 ulps of heading from +-y,
    where two atan2 implementations may land on different sides of the strict fold."""
    return name.startswith("heading_near_y")


def compare_to_oracle(got, scenes, max_objects, names=None):
    """got: dict objects / drone_index / n of a batch whose frame-set s is scenes[s].  Counts (clamped to max_objects),
    record order, drone_index, pos and error bit-exact; heading within HEADING_TOL, modulo pi for the scenes
    fold_allowed names.  Returns (objects compared, frame-sets truncated, worst heading difference)."""
    total, cut, worst = 0, 0, 0.0
    for s, (p, e) in enumerate(scenes):
        k, rec, di = oracle(p, e, max_objects)
        name = names[s] if names is not None else s
        assert got["n"][s] == k, (name, int(got["n"][s]), k)
        cut += oracle(p, e)[0] > max_objects
        if not k:
            continue
        g = got["objects"][s, :k]
        assert np.array_equal(got["drone_index"][s, :k], di), name
        assert np.array_equal(bits(g[:, :3]), bits(rec[:, :3])), name
        assert np.array_equal(bits(g[:, 4]), bits(rec[:, 4])), name
        dh = np.abs(g[:, 3] - rec[:, 3])
        if names is not None and fold_allowed(names[s]):
            dh = np.minimum(dh, np.abs(dh - np.pi))
        assert (dh <= HEADING_TOL).all(), (name, dh.max())
        worst = max(worst, float(dh.max()))
        total += k
    return total, cut, worst


def equal_but_heading(a, b, fold_sets=()):
    """Two runs of the same batch (the host build and the device): counts, drone_index, pos and error bit-equal over the
    valid records, heading within HEADING_TOL -- modulo pi in the frame-sets listed in fold_sets."""
    assert np.array_equal(a["n"], b["n"])
    valid = np.arange(a["objects"].shape[1])[None, :] < a["n"][:, None]
    assert np.array_equal(a["drone_index"][valid], b["drone_index"][valid])
    assert np.array_equal(bits(a["objects"][..., [0, 1, 2, 4]][valid]), bits(b["objects"][..., [0, 1, 2, 4]][valid]))
    dh = np.abs(a["objects"][..., 3] - b["objects"][..., 3])
    for s in fold_sets:
        dh[s] = np.minimum(dh[s], np.abs(dh[s] - np.pi))
    assert (dh[valid] <= HEADING_TOL).all(), dh[valid].max()
