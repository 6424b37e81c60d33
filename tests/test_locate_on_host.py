"""The drone locator's device code (csrc/locate_device.cuh) compiled for the host with g++, and the oracle it is held
to: RefPort.locate_objects equals the real reference's locate_objects on tests/golden/locate_edge.npz bit for bit, and
the host build equals the oracle on scenes that reach every branch of the greedy scan (tests/locate_util.py) -- counts,
record order, droneIndex, pos and error bit-exact, heading within 4 ulp of pi/2."""
import hashlib

import numpy as np
import pytest

from tests.locate_util import (D1, D2, GOLDEN, HEADING_TOL, MAX_POINTS, TOL, build_locate_host, compare_to_oracle, count_cases,
                               edge_scenes, equal_but_heading, fold_allowed, fuzz_scenes, golden_fuzz_scenes, host_locate,
                               host_locate_batch, large_scenes, oracle, pack, small_scenes, trace)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return build_locate_host(tmp_path_factory.mktemp("locate"))


# ---------------------------------------------------------------------------------------------- the oracle
def test_oracle_equals_the_reference_on_the_golden_scenes():
    """The named scenes and the fuzz sample are the ones the real reference was run on (points and errors bit-equal,
    the fuzz by digest), and RefPort.locate_objects gives its records: counts, order and droneIndex equal, pos / heading
    / error bit-equal."""
    z = np.load(GOLDEN)
    named = edge_scenes()
    assert list(z["names"]) == list(named)
    scenes = list(named.values()) + golden_fuzz_scenes()
    assert np.array_equal(z["n_points"], [len(p) for p, _ in scenes])
    edge = list(named.values())
    assert np.array_equal(z["edge_points"], np.concatenate([p for p, _ in edge]), equal_nan=True)
    assert np.array_equal(z["edge_errors"], np.concatenate([e for _, e in edge]))
    assert list(z["fuzz_sha256"]) == [hashlib.sha256(p.tobytes() + e.tobytes()).hexdigest() for p, e in scenes[len(edge):]]
    at = 0
    for s, (p, e) in enumerate(scenes):
        k, rec, di = oracle(p, e)
        assert k == z["n_objects"][s], s
        assert np.array_equal(rec.view(np.uint64), z["records"][at:at + k].view(np.uint64)), s
        assert np.array_equal(di, z["drone_index"][at:at + k]), s
        at += k
    assert at == len(z["records"]) > 9000 and len(scenes) - len(edge) == 300


def test_no_distance_lies_exactly_on_a_tolerance_edge():
    """The neighbour test is a strict < and the pair test refuses on a strict >, so the two treat |d - c| == 0.025
    differently -- but no double distance gets there: 0.095 and 0.15 are multiples of 2^-55, a distance between 0.0625
    and 0.25 is a multiple of 2^-56, so |d - c| is one too (the subtraction is exact), and the double 0.025 is an odd
    multiple of 2^-57.  The ulp scans of locate_util.tolerance_scenes therefore pin where each decision flips; which
    side equality falls on cannot be observed."""
    grid = 2.0 ** -56
    assert (0.025 / grid) % 1 == 0.5 and (D1 / grid) % 1 == 0 and (D2 / grid) % 1 == 0
    for lo, hi in ((D1 - TOL, D1 + TOL), (D2 - TOL, D2 + TOL)):
        assert 0.0625 < np.nextafter(lo, 0) and np.nextafter(hi, 1) < 0.25
        assert np.spacing(np.nextafter(lo, 0)) % grid == 0


# ---------------------------------------------------------------------------------------------- edge scenes
def _run(lib, scenes, R, max_objects):
    obj, err, n = pack(scenes, R)
    return host_locate(lib, obj, err, n, R, max_objects)


@pytest.mark.parametrize("R", [16, 64, MAX_POINTS])
def test_host_build_equals_the_oracle_on_the_edge_scenes(lib, R, capsys):
    """Every named scene that fits max_roots = R, one object slot per point.  The modulo-pi allowance on the heading is
    used by the "heading_near_y" scenes alone: their pair lies 1 .. 3 ulps of heading from +-y."""
    named = {k: v for k, v in edge_scenes().items() if len(v[0]) <= R}
    names = list(named)
    assert sum(map(fold_allowed, names)) == 12
    got = _run(lib, list(named.values()), R, R)
    total, cut, worst = compare_to_oracle(got, list(named.values()), R, names)
    with capsys.disabled():
        print(f"\nmax_roots {R}: {len(names)} edge scenes, {total} objects, worst heading difference {worst:.2e}")
    assert cut == 0 and total >= {16: 90, 64: 90, MAX_POINTS: 700}[R]


def test_edge_scenes_are_what_they_claim(lib):
    """On the host build: a pair along +-y heads exactly -+pi/2 (the strict folds leave it), along +-x and vertical 0;
    the apex at the pair's mean y gives droneIndex 1 and one ulp above it 0; the tolerance scans flip once each."""
    s = small_scenes()
    got = _run(lib, list(s.values()), 16, 16)
    at = {k: i for i, k in enumerate(s)}
    head = lambda k: got["objects"][at[k], 0, 3]
    assert head("heading_y_ab") == -np.pi / 2 and head("heading_y_ba") == np.pi / 2
    for k in ("heading_x_ab", "heading_x_ba", "heading_vertical_ab", "heading_vertical_ba"):
        assert got["n"][at[k]] == 1 and head(k) == 0.0
    for tag in ("ab", "ba"):
        assert all(abs(abs(head(f"heading_near_y_{k:+d}_{tag}")) - np.pi / 2) <= HEADING_TOL for k in (-3, -2, -1, 1, 2, 3))
    assert [int(got["drone_index"][at[f"index_{k:+d}ulp"], 0]) for k in (-1, 0, 1)] == [1, 1, 0]
    assert got["drone_index"][at["heading_vertical_ab"], 0] == 1          # apex y equals the pair's: not above it
    for scan in ("neighbour_0.070", "neighbour_0.120", "pair_0.125", "pair_0.175"):
        counts = [int(got["n"][at[f"{scan}_{k:+d}ulp"]]) for k in range(-8, 9)]
        assert sorted(set(counts)) == [0, 1] and sum(a != b for a, b in zip(counts, counts[1:])) == 1, (scan, counts)
    assert got["n"][at["empty"]] == got["n"][at["one_point"]] == got["n"][at["two_points"]] == 0


def test_scenes_reach_the_branches(capsys):
    """The large scenes share markers, have points with three and more neighbours, use rows >= 64 as i, a and b and
    skip matched rows >= 64; three place one triplet on rows that straddle 63 / 64 and use 127; the lattices come close
    to one object per point."""
    with capsys.disabled():
        print()
        for name, (p, e) in large_scenes().items():
            t = trace(p)
            assert len(t["triplets"]) == oracle(p, e)[0]
            print(f"{name}: {len(p)} points, {len(t['triplets'])} objects, {t['shared']} with an already matched marker, "
                  f"{t['many']} points with >= 3 neighbours, {t['high']} objects on rows >= 64, {t['screened_high']} rows >= 64 screened")
            if name.startswith(("crowded", "straddle")):
                assert t["shared"] >= 10 and t["many"] >= 40
            if len(p) == MAX_POINTS and not name.startswith("lattice"):
                assert t["high"] >= 20 and t["screened_high"] >= 10
    for name in ("straddle_63_64_127", "straddle_127_62_65", "straddle_64_0_127"):
        want = tuple(int(v) for v in name.split("_")[1:])
        assert want in trace(large_scenes()[name][0])["triplets"]
    p, e = large_scenes()["lattice_8x16"]
    assert oracle(p, e)[0] == 105


# ---------------------------------------------------------------------------------------------- counts, truncation
@pytest.mark.parametrize("R", [16, 64, MAX_POINTS])
def test_frame_set_counts(lib, R):
    """n_obj of 0, 1, 2, max_roots, max_roots + 5 and -1 over rows that hold valid triplets throughout: the locator
    reads min(n_obj, max_roots) rows and no others."""
    seen, (obj, err, n) = count_cases(R)
    assert list(n[:5]) == [0, 1, 2, R, R + 5] and n[6] == -1
    got = host_locate(lib, obj, err, n, R, R)
    total, _, _ = compare_to_oracle(got, seen, R)
    assert list(got["n"][[0, 1, 2, 6]]) == [0, 0, 0, 0] and got["n"][3] >= 1 and got["n"][4] == 1 and got["n"][5] == 1
    equal_but_heading(got, host_locate_batch(lib, obj, err, n, R, R))


@pytest.mark.parametrize("max_objects", [1, 3, 40])
def test_truncation_keeps_the_first_records_and_clamps_the_count(lib, max_objects):
    """More objects than max_objects: the first max_objects of the oracle's list, n == max_objects, and nothing
    written past them -- a sentinel slab after every frame-set's records and after the last one is untouched
    (host_locate checks it)."""
    named = edge_scenes()
    scenes = list(named.values())
    obj, err, n = pack(scenes, MAX_POINTS)
    got = host_locate(lib, obj, err, n, MAX_POINTS, max_objects)
    total, cut, _ = compare_to_oracle(got, scenes, max_objects, list(named))
    assert cut >= (9 if max_objects == 40 else 14)
    for s, (p, e) in enumerate(scenes):
        if oracle(p, e)[0] > max_objects:
            assert got["n"][s] == max_objects
    dense = host_locate_batch(lib, obj, err, n, MAX_POINTS, max_objects)
    for k in got:
        valid = np.arange(max_objects)[None, :] < got["n"][:, None]
        assert np.array_equal(got[k][valid] if k != "n" else got[k], dense[k][valid] if k != "n" else dense[k]), k


def test_frame_sets_are_independent(lib):
    """Permuting the frame-sets of a batch permutes the outputs, bit for bit."""
    scenes = list(edge_scenes().values())
    obj, err, n = pack(scenes, MAX_POINTS)
    a = host_locate_batch(lib, obj, err, n, MAX_POINTS, 48)
    perm = np.random.default_rng(7).permutation(len(scenes))
    b = host_locate_batch(lib, obj[perm], err[perm], n[perm], MAX_POINTS, 48)
    assert np.array_equal(a["n"][perm], b["n"])
    valid = np.arange(48)[None, :] < b["n"][:, None]
    assert np.array_equal(a["objects"][perm][valid].view(np.uint64), b["objects"][valid].view(np.uint64))
    assert np.array_equal(a["drone_index"][perm][valid], b["drone_index"][valid])


# ---------------------------------------------------------------------------------------------- fuzz
def test_host_build_equals_the_oracle_on_the_fuzz(lib, capsys):
    """2000 seeded scenes of 0-40 drones and 0-30 clutter points, jitter up to 0.02, with one object slot per point and
    with 4 slots.  Prints how many scenes reached what."""
    scenes = fuzz_scenes()
    obj, err, n = pack(scenes, MAX_POINTS)
    got = host_locate_batch(lib, obj, err, n, MAX_POINTS, MAX_POINTS)
    total, cut, worst = compare_to_oracle(got, scenes, MAX_POINTS)
    few = host_locate_batch(lib, obj, err, n, MAX_POINTS, 4)
    _, cut4, _ = compare_to_oracle(few, scenes, 4)
    stats = [trace(p) for p, _ in scenes]
    shared = sum(t["shared"] > 0 for t in stats); many = sum(t["many"] > 0 for t in stats)
    high = sum(t["high"] > 0 for t in stats); screened = sum(t["screened_high"] > 0 for t in stats)
    with capsys.disabled():
        print(f"\nfuzz: {len(scenes)} scenes, {total} objects, worst heading difference {worst:.2e}; scenes with a shared "
              f"marker {shared}, with a point of >= 3 neighbours {many}, with an object on rows >= 64 {high}, with a matched "
              f"row >= 64 screened {screened}, truncated at 4 objects {cut4}")
    assert cut == 0 and total > 40000
    assert min(shared, many) > 1200 and min(high, screened) > 400 and cut4 > 1200
