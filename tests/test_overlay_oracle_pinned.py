"""Pins tests/overlay_util.find_dot_drawn -- the oracle of the detection overlay -- against the real reference's
Cameras._find_dot (helpers.py:143-163), run unmodified where a checkout is named by MOCAP_REFERENCE_DIR.  CPU only."""
import numpy as np
import pytest

from oracle.ref_harness import load_reference, reference_available
from tests.overlay_util import find_dot_drawn, random_scene, sparse_scene

pytestmark = pytest.mark.skipif(not reference_available(), reason="needs the reference checkout (MOCAP_REFERENCE_DIR)")


def test_find_dot_drawing_equals_the_reference():
    """Random frames of every kind and size: the reference's drawn frame and points equal the oracle's."""
    _, cams = load_reference(4)
    rng = np.random.default_rng(17)
    for t in range(300):
        H, W = (int(v) for v in rng.integers(8, 160, 2))
        img = sparse_scene(rng, H, W, int(rng.integers(0, 20))) if t % 4 == 3 else random_scene(rng, H, W, ("noise", "blobs", "holes")[t % 3])
        got, pts = cams._find_dot(img.copy())
        want, want_pts = find_dot_drawn(img.copy())
        assert np.array_equal(got, want), t
        assert pts == (want_pts if want_pts else [[None, None]]), t


def _real_drawlines(helpers):
    """The reference's own drawlines (helpers.py:497-504), compiled from its source: the harness stubs it out."""
    import ast
    import cv2
    src = open(helpers.__file__).read()
    node = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "drawlines")
    ns = {"np": np, "cv": cv2}
    exec(compile(ast.Module(body=[node], type_ignores=[]), helpers.__file__, "exec"), ns)
    return ns["drawlines"]


def test_epipolar_lines_equal_the_reference_after_seeding():
    """The golden session's triangulating reads through the real find_point_correspondance_and_object_points, its real
    drawlines restored for this test, after np.random.seed(seed): the frames equal the oracle's lines in the colours of
    np.random.RandomState(seed).randint(0, 255, (L, 3)), the session's line counter carried from read to read."""
    from oracle.ref_port import RefPort
    from tests.live_util import DIST, K, TRIANGULATE, golden_scene, load_golden, render_read
    from tests.overlay_util import epilines_drawn, palette_of
    helpers, _ = load_reference(4, K)
    g = load_golden()
    scene = golden_scene(g)
    port = RefPort([K] * 4)
    stub = helpers.drawlines
    helpers.drawlines = _real_drawlines(helpers)
    try:
        seed, n = 11, 0
        np.random.seed(seed)
        palette = palette_of(seed, 4096)
        reads = 0
        for k in range(len(g["mode"])):
            if not int(g["mode"][k]) & TRIANGULATE or g["dark"][k]:
                continue
            raw = render_read(scene, k)
            frames = [port.preprocess(raw[c], c, DIST, scene["rotations"][c]) for c in range(4)]
            pts = [port.find_dot(f) for f in frames]
            want = [f.copy() for f in frames]
            got = [f.copy() for f in frames]
            helpers.find_point_correspondance_and_object_points([list(p) for p in pts], scene["poses"], got)
            n = epilines_drawn(port, want, pts, scene["poses"], palette, n)
            for c in range(4):
                assert np.array_equal(got[c], want[c]), (k, c)
            reads += 1
        assert reads > 50 and 200 < n < len(palette)
    finally:
        helpers.drawlines = stub
