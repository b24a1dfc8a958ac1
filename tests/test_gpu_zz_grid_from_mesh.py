"""GPU tests of the voxel grid from a mesh (i3d_grid_from_mesh, i3d_debug_get_grid_from_mesh_voxels) against the numpy restatement
tests/grid_from_mesh_ref.py.  Explicitly rounded arithmetic throughout: the bar is BYTE-EQUAL xyz and order, sdf0, sdf, weight, colour,
albedo, and the nearest face and feature per voxel."""
import os

import numpy as np
import pytest

import grid_from_mesh_ref as gr

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _engine():
    from intrinsic3d_b200.engine import Engine
    return Engine(0)


def _truth(name, n_theta=None):
    from intrinsic3d_b200.scene import config_geometry, truth_mesh
    return truth_mesh(n_theta, **config_geometry(name))


def _compare(e, n, r, voxel_size):
    g = e.download_grid()
    face, feat = e.debug_grid_from_mesh_voxels(n)
    assert n == len(r["xyz"]) and g["voxel_size"] == np.float32(voxel_size)
    assert g["xyz"].tobytes() == r["xyz"].tobytes()
    assert g["sdf0"].tobytes() == r["sdf"].tobytes() and g["sdf_refined"].tobytes() == r["sdf"].tobytes()
    assert (g["weight"] == 1.0).all() and (g["albedo"] == 0.6).all() and not g["rgb"].any()
    assert face.tobytes() == r["face"].tobytes() and feat.tobytes() == r["feature"].tobytes()
    return g


def _convert(e, mesh, vs, band, source="reference", cell=None):
    if source == "reference":
        e.upload_reference_mesh(mesh)
    n, info = e.grid_from_mesh(source, vs, band, cell)
    r = gr.grid_from_mesh(mesh, vs, band)
    _compare(e, n, r, vs)
    assert (info.num_voxels, info.num_negative, info.num_dropped_rim, info.num_dropped_zero_normal, info.num_dropped_zero_dot) == (
        n, r["num_negative"], r["num_dropped_rim"], r["num_dropped_zero_normal"], r["num_dropped_zero_dot"])
    assert (info.num_vertices_welded, info.num_boundary_edges) == (r["num_welded"], r["num_boundary_edges"])
    assert info.num_candidate_voxels == 512 * info.num_candidate_bricks >= n
    return n, info


def test_golden_fixture():
    g = np.load(os.path.join(HERE, "golden", "tiny_grid_from_mesh.npz"))
    e = _engine()
    e.upload_reference_mesh(dict(vertices=g["vertices"], faces=g["faces"]))
    n, _ = e.grid_from_mesh("reference", float(g["voxel_size"]), float(g["band"]))
    _compare(e, n, dict(xyz=g["xyz"], sdf=g["sdf"], face=g["face"], feature=g["feature"]), float(g["voxel_size"]))


MESHES = {
    "cube": lambda: gr.box_mesh([-0.043, -0.031, -0.0275], [0.041, 0.052, 0.0385]),
    "cube_rotated_split": lambda: gr.split_vertices(gr.box_mesh([-0.04, -0.03, -0.035], [0.045, 0.05, 0.03], gr.np.array(
        [[0.36, -0.48, 0.8], [0.8, 0.6, 0.0], [-0.48, 0.64, 0.6]]), np.array([0.0013, -0.0021, 0.0007]))),
    "l_prism": lambda: gr.l_prism(0.04, np.array([-0.0312, -0.0287, -0.0193]))[0],
    "wedge": lambda: gr.wedge(0.08, 25.0, 0.05, np.array([-0.0412, -0.0037, -0.0231]))[0],
    "patch": lambda: gr.square_patch(-0.0405, 0.0395, 0.00337, 3),
}


@pytest.mark.parametrize("band", [1.0, 3.0, 5.0])
@pytest.mark.parametrize("name", sorted(MESHES))
def test_meshes(name, band):
    e = _engine()
    _convert(e, MESHES[name](), 0.01, band)


def test_tiny_small_and_both_sources(tiny_scene, small_scene):
    for s, name in ((tiny_scene, "tiny"), (small_scene, "small")):
        vs = float(s["voxel_size"])
        e = _engine()
        e.load_scene(s)
        _convert(e, _truth(name, 64 if name == "tiny" else None), vs, 3.0)
        e.load_scene(s)
        m = e.extract_mesh("fused", False)
        _convert(e, m, vs, 3.0, source="resident")


def test_c2():
    e = _engine()
    n, info = _convert(e, _truth("c2", 256), 0.002, 3.0)
    print("c2", n, info.as_dict())


def test_independent_of_the_cell_size(tiny_scene):
    e = _engine()
    e.upload_reference_mesh(_truth("tiny", 64))
    res = []
    for cell in (None, 0.7 * 0.004, 5.0 * 0.004):
        n, info = e.grid_from_mesh("reference", 0.004, 3.0, cell)
        g = e.download_grid()
        res.append((info.cell_size, g["xyz"].tobytes(), g["sdf0"].tobytes(), e.debug_grid_from_mesh_voxels(n)[0].tobytes()))
    assert len({r[0] for r in res}) == 3
    assert all(r[1:] == res[0][1:] for r in res)


def test_c3_run_to_run():
    e = _engine()
    e.upload_reference_mesh(_truth("c3"))
    out = []
    for _ in range(2):
        n, info = e.grid_from_mesh("reference", 0.002, 3.0)
        g = e.download_grid()
        out.append((g["xyz"].tobytes(), g["sdf0"].tobytes(), e.debug_grid_from_mesh_voxels(n)[1].tobytes()))
        print("c3", n, {k: v for k, v in info.as_dict().items() if k.startswith(("ms_", "num_candidate", "point"))})
    assert out[0] == out[1]


# measured on an H100 80GB HBM3 (tiny scene, L = 2): mean 0.0097 / 0.0098 voxel and max 0.062 / 0.059 voxel (accuracy / completeness);
# the bounds are about twice that
ROUND_TRIP_MEAN, ROUND_TRIP_MAX = 0.02, 0.12          # voxels


def test_round_trip(tiny_scene):
    s = tiny_scene
    vs = float(s["voxel_size"])
    e = _engine()
    e.load_scene(s)
    m0 = e.extract_mesh("fused", False)
    e.grid_from_mesh("resident", vs, 3.0)
    g1 = e.download_grid()
    m1 = e.extract_mesh("fused", False)
    e.upload_reference_mesh(m0)
    d = e.surface_distance((0.1 * vs,), 2 * vs, 2)
    print("round trip", {k: d["accuracy"][k] / vs for k in ("mean", "max")}, {k: d["completeness"][k] / vs for k in ("mean", "max")})
    for side in ("accuracy", "completeness"):
        assert d[side]["num_matched"] == d[side]["num_samples"]
        assert d[side]["mean"] <= ROUND_TRIP_MEAN * vs and d[side]["max"] <= ROUND_TRIP_MAX * vs
    assert len(m1["faces"]) > 0
    # converting the same mesh again, on another engine, gives the same bytes
    e2 = _engine()
    e2.load_scene(s)
    e2.extract_mesh("fused", False)
    e2.grid_from_mesh("resident", vs, 3.0)
    g2 = e2.download_grid()
    assert g1["xyz"].tobytes() == g2["xyz"].tobytes() and g1["sdf0"].tobytes() == g2["sdf0"].tobytes()


def test_refinement_runs_on_a_converted_grid(small_scene):
    from intrinsic3d_b200.ctypes_defs import default_params
    from intrinsic3d_b200.engine import default_lighting_params
    from intrinsic3d_b200.scene import make_color_frames
    s = small_scene
    vs = float(s["voxel_size"])
    e = _engine()
    e.load_scene(s)
    e.upload_color_frames(make_color_frames(s))
    e.upload_reference_mesh(_truth("small"))
    n, _ = e.grid_from_mesh("reference", vs, 3.0)
    rec, obs = e.recompute_colors()
    assert rec > 0.5 * n and obs > 0
    lp = default_lighting_params()
    lp.thres_shell = s["thres_shell"]
    li = e.estimate_lighting(lp)
    assert li.num_subvolumes > 0
    p = default_params()
    p.thres_shell = s["thres_shell"]
    p.forced_cg_iterations = 4
    for _ in range(2):
        it = e.gn_iteration(p)
        assert np.isfinite(it.cost_final) and it.cost_final <= it.cost_initial
    m = e.clear_voxels_outside_thin_shell(s["thres_shell"])
    assert 0 < m <= n
    assert e.upsample_grid() > m
    assert len(e.extract_mesh("refined", False)["faces"]) > 0


def test_refusals_change_nothing(tiny_scene):
    import ctypes as C
    from intrinsic3d_b200.engine import default_fusion_params
    from intrinsic3d_b200.ctypes_defs import I3DGridFromMeshParams
    s = tiny_scene
    vs = float(s["voxel_size"])
    e = _engine()
    e.load_scene(s)
    truth = _truth("tiny", 64)
    e.upload_reference_mesh(truth)
    e.grid_from_mesh("reference", vs, 3.0)
    face0 = e.debug_grid_from_mesh_voxels(e.n)
    m = e.extract_mesh("refined", False)
    fp = default_fusion_params()
    fp.voxel_size = vs
    e.fusion_begin(fp)

    def state():
        g = e.download_grid()
        mm = e._download_mesh(m["info"])
        return [g[k].tobytes() for k in ("xyz", "sdf0", "sdf_refined", "albedo", "weight", "rgb")] + [mm[k].tobytes() for k in ("vertices", "faces")] + [
            e.fusion_volume()["xyz"].tobytes()] + [a.tobytes() for a in e.debug_grid_from_mesh_voxels(len(face0[0]))]
    before = state()
    bad = [dict(voxel_size=0.0), dict(voxel_size=float("nan")), dict(band=0.0), dict(band=16.5), dict(cell_size=-1.0), dict(cell_size=float("inf")),
           dict(voxel_size=1e-9), dict(source=7)]
    for kw in bad:
        prm = I3DGridFromMeshParams(kw.get("source", 0), kw.get("voxel_size", vs), kw.get("band", 3.0), kw.get("cell_size", 0.0))
        assert e.L.i3d_grid_from_mesh(e.h, C.byref(prm), None) != 0, kw
        assert state() == before, kw
    # no voxel: a tiny face between lattice points, with a band narrower than its distance to the nearest one
    e2 = _engine()
    e2.load_scene(s)
    e2.upload_reference_mesh(dict(vertices=np.array([[0.0015, 0.0015, 0.0015], [0.0016, 0.0015, 0.0015], [0.0015, 0.0016, 0.0015]], np.float32),
                                  faces=np.array([[0, 1, 2]], np.int32)))
    g0 = e2.download_grid()
    with pytest.raises(RuntimeError, match="no voxel"):
        e2.grid_from_mesh("reference", 0.004, 0.1)
    assert e2.download_grid()["sdf0"].tobytes() == g0["sdf0"].tobytes()
    # the reference mesh is unchanged: converting it again gives the first grid
    e.grid_from_mesh("reference", vs, 3.0)
    assert e.debug_grid_from_mesh_voxels(len(face0[0]))[0].tobytes() == face0[0].tobytes()
