"""The TSDF host model (tests/tsdf_f32.py) and the mesh PLY writer, without a GPU: the derived triangle table, the model
against analytic surfaces, and the PLY layout."""
import numpy as np
import pytest

import tsdf_f32 as m
import tsdf_scenes as ts


def fuse(sc, thr=3.0):
    grid = {}
    for v in sc.views:
        cam = m.Camera(v.K, v.E, *v.depth.shape, sc.vs, sc.depth_scale, sc.depth_max, sc.trunc_mult)
        m.integrate(grid, cam, m.touch(cam, v.depth), v.depth, v.color)
    verts, cols, tris = m.extract(grid, sc.vs, thr)
    return grid, verts, cols, tris


def manifold_report(verts, tris):
    """(boundary edges, edges not shared by exactly two triangles, Euler characteristic, signed volume)"""
    e = np.sort(np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]]), axis=1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    v = verts.astype(np.float64)
    vol = np.einsum("ij,ij->i", v[tris[:, 0]], np.cross(v[tris[:, 1]], v[tris[:, 2]])).sum() / 6
    return int((cnt == 1).sum()), int((cnt != 2).sum()), len(verts) - len(cnt) + len(tris), vol


# ---- the table ----------------------------------------------------------------------------------------------------------

def _sign_change_edges(case):
    ins = [(case >> c) & 1 for c in range(8)]
    return {e for e in range(12) if ins[m.corner_id(m.edge_ends(e)[0])] != ins[m.corner_id(m.edge_ends(e)[1])]}


def test_table_loops_are_closed_and_cover_every_sign_change_edge_once():
    for case in range(256):
        lps = m.loops(case)
        used = [e for lp in lps for e in lp]
        assert sorted(used) == sorted(_sign_change_edges(case)), case      # each sign-change edge in exactly one loop
        succ, _ = m.face_segments(case)
        for lp in lps:
            assert len(lp) >= 3 and all(succ[lp[k]] == lp[(k + 1) % len(lp)] for k in range(len(lp)))   # closed
            assert lp[0] == min(lp)                                          # fanned from its lowest edge
        tris = m.TABLE[case]
        assert len(tris) == sum(len(lp) - 2 for lp in lps) and {e for t in tris for e in t} == _sign_change_edges(case)
    assert m.TABLE[0] == [] and m.TABLE[255] == [] and m.TABLE[1] == [(0, 4, 8)]


def test_complementary_cases_have_opposite_winding():
    """On every face that is not ambiguous, the complementary case has the same segment, reversed; with no ambiguous face at
    all the whole loop set is reversed."""
    for case in range(256):
        s1, amb1 = m.face_segments(case)
        s2, amb2 = m.face_segments(255 - case)
        assert amb1 == amb2
        for a, b in s1.items():
            on_ambiguous = any(e // 4 != ax and m.edge_ends(e)[0][ax] == sd for e in (a, b) for ax, sd in amb1 if
                               all(x // 4 != ax and m.edge_ends(x)[0][ax] == sd for x in (a, b)))
            if not on_ambiguous:
                assert s2[b] == a, (case, a, b)


def test_table_winding_points_to_increasing_tsdf():
    """With a linear field f = g . (p - p0) crossing the cube (no ambiguous face), the right-hand normal of every triangle
    points along the gradient g (toward increasing tsdf)."""
    rng = np.random.default_rng(0)
    hit = set()
    for _ in range(3000):
        g = rng.normal(size=3)
        f = (m.CORNERS - rng.uniform(0.2, 0.8, 3)) @ g
        case = int(sum(1 << c for c in range(8) if f[c] < 0))
        if case in (0, 255):
            continue
        hit.add(case)
        pts = {}
        for e in range(12):
            p, q = m.edge_ends(e)
            f0, f1 = f[m.corner_id(p)], f[m.corner_id(q)]
            if (f0 < 0) != (f1 < 0):
                pts[e] = p + f0 / (f0 - f1) * (q - p)
        for a, b, c in m.TABLE[case]:
            n = np.cross(pts[b] - pts[a], pts[c] - pts[a])
            assert np.dot(n, g) > -1e-12, case
    assert len(hit) > 20


# ---- the model against analytic surfaces ---------------------------------------------------------------------------------

def test_fronto_plane():
    """Camera at the origin looking down +z at the plane z = D: every updated voxel holds min(D - z, trunc) / trunc up to fp32
    rounding, and every vertex lies on the plane."""
    sc = ts.make("fronto")
    sc.views = sc.views[:1] * 3               # the same plane three times: weight 3 reaches the threshold
    D = float(sc.views[0].depth[0, 0])
    assert np.all(sc.views[0].depth == np.float32(D))
    grid, verts, cols, tris = fuse(sc)
    keys, tsdf, w, _ = m.active(grid)
    g = m.grid_points(m.unpack(keys))
    z = g[..., 2] * np.float64(np.float32(sc.vs))
    trunc = float(np.float32(np.float32(8.0) * np.float32(sc.vs)))
    upd = w > 0
    want = np.minimum(D - z, trunc) / trunc
    assert upd.sum() > 1000 and np.abs(tsdf[upd] - want[upd]).max() < 4e-6
    assert np.all(want[upd] >= -1.0)
    assert len(tris) > 100 and np.abs(verts[:, 2] - D).max() < 2e-6


def test_sphere_from_all_around_is_watertight_and_close():
    """Bound, stated before the run.  Each view's projective distance d - z_c has its zero on the sphere up to the depth change
    across one pixel (footprint (dist + r) / f, times a slope of at most 2 inside the band), and linear interpolation of a
    field with curvature 1/r across one voxel moves the crossing by at most vs^2 / (8 r).  Views that see a voxel at a grazing
    angle contribute clipped (min(sdf, trunc)) or one-sided values; that bias keeps the crossing within half the truncation
    band.  So  bound = 2 (dist + r) / f + vs^2 / (8 r) + trunc / 2.  The band is 4 voxels here: with 8, single grazing views
    leave small closed bubbles just outside the surface (the mesh stays closed, but is no longer one sphere)."""
    r, dist, vs, W = 0.3, 1.2, 0.02, 96
    sc = ts.sphere_scene(30, W, 80, vs=vs, r=r, dist=dist)
    sc.trunc_mult = 4.0
    f = sc.views[0].K[0, 0]
    bound = 2 * (dist + r) / f + vs * vs / (8 * r) + sc.trunc_mult * vs / 2
    _, verts, _, tris = fuse(sc)
    boundary, bad, chi, vol = manifold_report(verts, tris)
    assert len(tris) > 500
    assert boundary == 0 and bad == 0 and chi == 2 and vol > 0
    err = np.abs(np.linalg.norm(verts.astype(np.float64), axis=1) - r)
    assert err.max() < bound, (err.max(), bound)


def test_normals_model_zero_sum_and_order():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 5]], np.float32)
    t = np.array([[0, 1, 2], [0, 2, 1]], np.int32)         # opposite faces cancel: zero sum, no NaN
    n = m.vertex_normals(v, t)
    assert np.array_equal(n, np.zeros((4, 3), np.float32))
    n = m.vertex_normals(v, t[:1])
    assert np.array_equal(n[:3], np.tile(np.float32([0, 0, 1]), (3, 1))) and np.array_equal(n[3], np.zeros(3, np.float32))


# ---- PLY ---------------------------------------------------------------------------------------------------------------

def test_mesh_ply_layout_and_round_trip(tmp_path):
    from rade_gs_b200.ply_io import read_ply_vertices, save_triangle_mesh_ply
    rng = np.random.default_rng(1)
    v = rng.normal(size=(7, 3)).astype(np.float32)
    n = rng.normal(size=(7, 3)).astype(np.float32)
    c = np.array([[0, 1, 0.5], [-0.2, 1.7, 0.498], [0.002, 0.999, 0.5 + 1 / 510]] + [[0.25, 0.75, 1.0]] * 4, np.float32)
    t = rng.integers(0, 7, (5, 3)).astype(np.int32)
    p = tmp_path / "mesh.ply"
    save_triangle_mesh_ply(str(p), v, t, c, n)
    raw = p.read_bytes()
    head = raw[:raw.index(b"end_header\n") + len(b"end_header\n")]
    assert head.decode().split("\n")[:-1] == [
        "ply", "format binary_little_endian 1.0", "element vertex 7", "property float x", "property float y", "property float z",
        "property float nx", "property float ny", "property float nz", "property uchar red", "property uchar green", "property uchar blue",
        "element face 5", "property list uchar int vertex_indices", "end_header"]
    body = raw[len(head):]
    assert len(body) == 7 * (24 + 3) + 5 * (1 + 12)
    vd = np.dtype([("p", "<f4", 6), ("c", "u1", 3)])
    vert = np.frombuffer(body[:7 * 27], vd)
    assert np.array_equal(vert["p"][:, :3], v) and np.array_equal(vert["p"][:, 3:], n)
    assert np.array_equal(vert["c"], np.floor(255 * np.clip(c.astype(np.float64), 0, 1) + 0.5).astype(np.uint8))
    assert vert["c"][0].tolist() == [0, 255, 128] and vert["c"][1].tolist() == [0, 255, 127]
    face = np.frombuffer(body[7 * 27:], np.dtype([("n", "u1"), ("i", "<i4", 3)]))
    assert np.all(face["n"] == 3) and np.array_equal(face["i"], t)
    props = read_ply_vertices(str(p))
    assert np.array_equal(props["x"], v[:, 0]) and np.array_equal(props["blue"], vert["c"][:, 2])


def test_mesh_ply_without_normals_or_colours(tmp_path):
    from rade_gs_b200.ply_io import save_triangle_mesh_ply
    p = tmp_path / "m.ply"
    save_triangle_mesh_ply(str(p), np.zeros((3, 3), np.float32), np.array([[0, 1, 2]], np.int32))
    raw = p.read_bytes()
    assert raw.endswith(bytes([3]) + np.array([0, 1, 2], "<i4").tobytes())
    assert len(raw) - raw.index(b"end_header\n") - 11 == 3 * 27 + 13
