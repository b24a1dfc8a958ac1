"""CPU tests of the mesh colour modes: known answers for the numpy restatement tests/vis_ref.py, the committed fixture, and the host
helpers of intrinsic3d_b200/mesh.py (output_modes, export_meshes).  The device kernels are checked against vis_ref in
tests/test_gpu_zz_vis.py."""
import os

import numpy as np
import pytest

import vis_ref
from intrinsic3d_b200 import mesh

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32


def box(shape, sdf_fn, weight=None, rgb=None, albedo=0.6, voxel_size=0.25, drop=()):
    """A dense box of voxels 0..shape-1 with sdf_fn(x, y, z) (float64) as both sdf0 and refined sdf; `drop` removes coordinates."""
    c = np.stack(np.meshgrid(*[np.arange(s) for s in shape], indexing="ij"), -1).reshape(-1, 3)
    keep = np.array([tuple(p) not in set(drop) for p in c], bool)
    c = c[keep]
    n = len(c)
    sdf = np.asarray(sdf_fn(c[:, 0], c[:, 1], c[:, 2]), np.float64) * np.ones(n)
    g = dict(xyz=c.astype(np.int32), sdf0=sdf.copy(), sdf_refined=sdf, albedo=np.broadcast_to(np.asarray(albedo, np.float64), (n,)).copy(),
             weight=np.ones(n, np.float32), rgb=np.full((n, 3), 100, np.uint8), voxel_size=F32(voxel_size))
    if weight is not None:
        for p, w in weight.items():
            g["weight"][_at(g, p)] = w
    if rgb is not None:
        g["rgb"][:] = rgb
    return g


def _at(g, p):
    return int(np.flatnonzero((g["xyz"] == np.asarray(p)).all(1))[0])


def test_planar_sdf_normals_and_laplacian():
    for sign, want in ((1.0, (255, 127, 127)), (-1.0, (0, 127, 127))):
        g = box((5, 5, 5), lambda x, y, z: sign * 0.25 * (x - 2.0))
        nrm = vis_ref.colors(g, "normals")
        assert tuple(nrm[_at(g, (2, 2, 2))]) == want
        assert tuple(nrm[_at(g, (4, 2, 2))]) == (0, 0, 0)          # no +x neighbour: zero normal
        lap = vis_ref.colors(g, "lap")
        assert tuple(lap[_at(g, (2, 2, 2))]) == (127, 127, 127)    # linear sdf: Laplacian 0 -> 0.5 * 255 truncated
        assert tuple(lap[_at(g, (0, 2, 2))]) == (0, 0, 0)          # -x neighbour missing
    # the normals along y and z, and a diagonal plane with an inexact normal, truncated per channel
    g = box((5, 5, 5), lambda x, y, z: -0.25 * (z - 2.0))
    assert tuple(vis_ref.colors(g, "normals")[_at(g, (2, 2, 2))]) == (127, 127, 0)
    g = box((5, 5, 5), lambda x, y, z: 0.25 * (x + y))
    c = vis_ref.colors(g, "normals")[_at(g, (2, 2, 2))]
    n = F32(0.25) / np.sqrt(F32(0.25) * F32(0.25) + F32(0.25) * F32(0.25))
    v = (F32(0.5) * n + F32(0.5)) * F32(255)
    assert tuple(c) == (int(v), int(v), 127) and int(v) == 217


def test_laplacian_known_value():
    # sdf = x^2 / 8 (exact floats): dxx = 2/8 = 0.25 everywhere; truncation 5 * 0.25 -> lap 0.2f -> (0.1 + 0.5) * 255 = 153.00001f
    g = box((5, 5, 5), lambda x, y, z: (x - 2.0) ** 2 / 8.0)
    lap = vis_ref.colors(g, "lap")[_at(g, (2, 2, 2))]
    l = F32(0.25) / (F32(0.25) * F32(5))
    assert lap[0] == int((F32(0.5) * l + F32(0.5)) * F32(255)) == 153


def test_albedo_and_truncation():
    g = box((2, 2, 2), lambda x, y, z: 0.0 * x)
    g["albedo"][:] = [0.6, np.nextafter(0.6, 0.0), 0.0, -0.5, 1.0, 2.0, 1.0 / 255.0, 0.999]
    c = vis_ref.colors(g, "albedo")[:, 0]
    assert c.tolist() == [153, 152, 0, 0, 255, 255, 1, 254]


def test_intensity_edges():
    assert (F32(0.299) * F32(255) + F32(0.587) * F32(255)) + F32(0.114) * F32(255) == F32(255)
    g = box((2, 2, 2), lambda x, y, z: 0.0 * x)
    g["rgb"][:] = [[255, 255, 255], [0, 0, 0], [1, 0, 0], [0, 0, 9], [10, 10, 10], [3, 3, 3], [0, 255, 0], [255, 0, 0]]
    lum = vis_ref.intensity(g["rgb"])
    c = vis_ref.colors(g, "lum")
    assert c[0].tolist() == [255, 255, 255] and c[1].tolist() == [0, 0, 0]
    assert (c[:, 0] == np.floor(lum).astype(np.uint8)).all()
    # a grey whose float intensity lies just below the integer truncates to the integer below it
    greys = np.arange(256)
    li = vis_ref.intensity(np.repeat(greys[:, None], 3, 1).astype(np.uint8))
    below = greys[li < greys]
    assert len(below) > 0
    gb = box((1, 1, 1), lambda x, y, z: 0.0 * x, rgb=[below[0]] * 3)
    assert vis_ref.colors(gb, "lum")[0, 0] == below[0] - 1


def test_intensity_gradient_and_ring():
    g = box((4, 3, 3), lambda x, y, z: 0.0 * x)
    for i, p in enumerate(g["xyz"]):
        g["rgb"][i] = [40 * p[0], 0, 0]
    c = vis_ref.colors(g, "lum_grad")
    v = (F32(0.299) * F32(80) - F32(0.299) * F32(40)) * F32(0.5) + F32(127)
    assert c[_at(g, (1, 1, 1))].tolist() == [int(v)] * 3
    assert c[_at(g, (0, 1, 1))].tolist() == [127] * 3              # missing -x neighbour
    # a zero-weight ring neighbour invalidates the ring (the voxel itself need not be valid for lap / lum_grad)
    g2 = box((4, 3, 3), lambda x, y, z: 0.0 * x, weight={(1, 1, 2): 0.0, (2, 1, 1): 0.0})
    g2["rgb"][:] = g["rgb"]
    assert vis_ref.colors(g2, "lum_grad")[_at(g2, (1, 1, 1))].tolist() == [127] * 3
    assert vis_ref.colors(g2, "lap")[_at(g2, (1, 1, 1))].tolist() == [0] * 3
    assert vis_ref.colors(g2, "lap")[_at(g2, (2, 1, 1))].tolist() == [127] * 3      # invalid itself, valid ring
    # clamping at both ends
    g3 = box((3, 3, 3), lambda x, y, z: 0.0 * x)
    g3["rgb"][_at(g3, (2, 1, 1))] = [255, 255, 255]
    g3["rgb"][_at(g3, (1, 1, 1))] = [0, 0, 0]
    assert vis_ref.colors(g3, "lum_grad")[_at(g3, (1, 1, 1))].tolist() == [254] * 3   # 255 * 0.5 + 127 = 254.5
    g3["rgb"][:] = 255
    g3["rgb"][_at(g3, (2, 1, 1))] = [0, 0, 0]
    assert vis_ref.colors(g3, "lum_grad")[_at(g3, (1, 1, 1))].tolist() == [0] * 3


def test_chromacity():
    g = box((2, 2, 2), lambda x, y, z: 0.0 * x)
    g["rgb"][:] = [[10, 10, 10], [200, 200, 200], [0, 0, 0], [255, 0, 0], [1, 1, 1], [0, 0, 1], [100, 50, 25], [255, 255, 255]]
    c = vis_ref.colors(g, "chroma")
    for i in (0, 1, 4, 7):
        assert c[i].tolist() == [127, 127, 127]                        # grey: chromacity 1 -> 127.5 truncated
    assert c[2].tolist() == [0, 0, 0]
    assert c[3].tolist() == [255, 0, 0]                                # 1 / 0.299 * 127.5 clamps at 255
    lum = F32(0.114)
    assert c[5].tolist() == [0, 0, 255] and F32(1) / lum * F32(127.5) > 255


def test_shading_single_subvolume_and_zero_normal():
    # sdf along z: normal (0, 0, 1), basis (1, 0, 1, 0, 0, 0, 2, 0, 0)
    g = box((3, 3, 3), lambda x, y, z: 0.25 * z, albedo=0.5)
    sh = np.array([[0.3, 0.1, 0.2, 0.0, 0.0, 0.0, 0.05, 0.0, 0.0]])
    idx = np.zeros((1, 3), np.int32)
    c = vis_ref.colors(g, "shading_sv", sub_index=idx, sub_sh=sh, subvolume_size=100.0)
    s32 = sh[0].astype(F32)
    d = ((s32[0] * F32(1) + s32[2] * F32(1)) + s32[6] * F32(2))
    want = int(F32(float(F32(0.5) * d) * 255.0))
    assert c[_at(g, (1, 1, 1))].tolist() == [want] * 3
    cc = vis_ref.colors(g, "shading_sv_const", sub_index=idx, sub_sh=sh, subvolume_size=100.0)
    assert cc[_at(g, (1, 1, 1))].tolist() == [int(F32(float(F32(0.7) * d) * 255.0))] * 3
    assert c[_at(g, (1, 1, 2))].tolist() == [0, 0, 0]                  # no +z neighbour: zero normal
    # one subvolume: its SH is used as it is, even where the blend would find no subvolume around the voxel
    far = vis_ref.colors(g, "shading_sv", sub_index=np.array([[50, 50, 50]], np.int32), sub_sh=sh, subvolume_size=0.01)
    assert (far == c).all()
    # albedo 0 gives 0; a constant sdf (zero normal) gives 0
    g["albedo"][:] = 0.0
    assert (vis_ref.colors(g, "shading_sv", sub_index=idx, sub_sh=sh, subvolume_size=100.0) == 0).all()
    g0 = box((3, 3, 3), lambda x, y, z: 0.0 * x)
    assert (vis_ref.colors(g0, "shading_sv_const", sub_index=idx, sub_sh=sh, subvolume_size=100.0) == 0).all()


def test_shading_blend_branch():
    # two subvolumes of size 1 m along x (voxel size 0.25 m: 4 voxels each); the blend between them is linear in x
    g = box((8, 3, 3), lambda x, y, z: 0.25 * z, albedo=1.0)
    idx = np.array([[0, 0, 0], [1, 0, 0]], np.int32)
    sh = np.zeros((2, 9))
    sh[0, 0], sh[1, 0] = 0.2, 0.6
    blended = vis_ref.blend_sh(g["xyz"], g["voxel_size"], idx, sh, 1.0)
    x = g["xyz"][:, 0]
    # voxel x at p = 0.25 x m -> subvolume coordinate 0.25 x - 0.5: below 0.5 only cell 0 (and the missing cell -1), above 1.5 only cell 1
    assert np.allclose(blended[x <= 2, 0], 0.2) and np.allclose(blended[x >= 6, 0], 0.6)
    mid = (x > 2) & (x < 6)
    assert np.allclose(blended[mid, 0], 0.2 + 0.4 * (0.25 * x[mid] - 0.5 - 0.0))
    c = vis_ref.colors(g, "shading_sv", sub_index=idx, sub_sh=sh, subvolume_size=1.0)
    sh_f = blended.astype(F32)
    ok = (g["xyz"] < [7, 2, 2]).all(1)                                 # the voxels with a +x, +y and +z neighbour
    want = (sh_f[:, 0] * F32(1) + sh_f[:, 2] * F32(1)) + sh_f[:, 6] * F32(2)
    want = np.trunc(((F32(1) * want).astype(np.float64) * 255.0).astype(F32)).astype(np.uint8)
    assert (c[ok, 0] == want[ok]).all() and (c[~ok] == 0).all()
    # no subvolume around the voxels at all: SH 0 -> black
    far = vis_ref.colors(g, "shading_sv", sub_index=idx + 100, sub_sh=sh, subvolume_size=1.0)
    assert (far == 0).all()


def test_golden_fixture():
    f = np.load(os.path.join(HERE, "golden", "tiny_vis.npz"))
    g = {k: f[k] for k in ("xyz", "sdf0", "sdf_refined", "albedo", "weight", "rgb", "voxel_size")}
    assert f["sub_sh"].shape[0] > 1
    for src in ("fused", "refined"):
        for mode in vis_ref.MODES:
            c = vis_ref.colors(g, mode, src, f["sub_index"], f["sub_sh"], float(f["subvolume_size"]))
            assert c.tobytes() == f[f"{src}_{mode or 'voxel'}"].tobytes(), (src, mode)
    # the fixture exercises every branch: refined differs from fused, the albedo varies, the modes differ from the voxel colours
    assert not np.array_equal(g["sdf0"], g["sdf_refined"]) and len(np.unique(g["albedo"])) > 10
    assert len({f[f"refined_{m or 'voxel'}"].tobytes() for m in vis_ref.MODES}) == len(vis_ref.MODES)


YML = {  # data/intrinsic3d.yml as shipped (the visualisation keys)
    "output_mesh_normals": "0", "output_mesh_laplacian": "0", "output_mesh_intensity": "0", "output_mesh_intensity_grad": "0",
    "output_mesh_albedo": "1", "output_mesh_shading_sv": "0", "output_mesh_shading_sv_const": "0", "output_mesh_chromacity": "0",
    "output_mesh_subvolumes": "0", "output_mesh_subvolumes_interpolated": "0", "output_mesh_largest_comp_only": "1",
}


def test_output_modes():
    assert mesh.output_modes(YML) == ["", "albedo"]
    assert mesh.output_modes(YML, add_voxel_colors=False) == ["albedo"]
    on = {k: "1" for k in YML}
    assert mesh.output_modes(on) == ["", "normals", "lap", "lum", "lum_grad", "albedo", "shading_sv", "shading_sv_const", "chroma", "subvol",
                                     "subvol_interp"]
    assert mesh.output_modes({}) == [""]                                        # absent keys add nothing
    assert mesh.output_modes({"output_mesh_chromacity": 1, "output_mesh_normals": True, "output_mesh_lap": "1"}) == ["", "normals", "chroma"]


class _FakeEngine:
    def __init__(self):
        self.calls = []

    def extract_mesh(self, source, largest_component_only, color_mode):
        self.calls.append((source, largest_component_only, color_mode))
        return dict(vertices=np.zeros((3, 3), np.float32), colors=np.full((3, 3), len(self.calls), np.uint8), faces=np.array([[0, 1, 2]], np.int32))


def test_export_meshes_file_names(tmp_path):
    e = _FakeEngine()
    prefix = str(tmp_path / "mesh")
    paths = mesh.export_meshes(e, prefix, ["", "albedo", "shading_sv"], True)
    assert paths == [prefix + ".ply", prefix + "_albedo.ply", prefix + "_shading_sv.ply"]
    assert e.calls == [("refined", True, ""), ("refined", True, "albedo"), ("refined", True, "shading_sv")]
    for i, p in enumerate(paths):
        assert open(p, "rb").read() == mesh.ply_bytes(dict(vertices=np.zeros((3, 3), np.float32), colors=np.full((3, 3), i + 1, np.uint8),
                                                           faces=np.array([[0, 1, 2]], np.int32)))
    # the subvolume modes are refused before anything is written
    e2 = _FakeEngine()
    with pytest.raises(ValueError, match="subvol"):
        mesh.export_meshes(e2, str(tmp_path / "other"), ["", "subvol"], False)
    assert e2.calls == [] and not os.path.exists(str(tmp_path / "other.ply"))
