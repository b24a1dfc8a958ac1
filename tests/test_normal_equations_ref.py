"""CPU checks of the float64 normal-equation reference (tests/normal_equations_ref.py) before it judges any GPU kernel:
built from the oracle's own rows and Jacobian it reproduces the oracle's Jacobi column scale, and its componentwise comparator
flags small deliberate errors (a dropped row, a double-added warp partial, a column off by 1e-5)."""
import numpy as np
import pytest

import normal_equations_ref as ner


def _params(scene, **kw):
    from intrinsic3d_b200.ctypes_defs import default_params
    p = default_params()
    p.thres_shell = scene["thres_shell"]
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.fixture(scope="module")
def oracle_rows(tiny_scene):
    from oracle import Oracle
    s = tiny_scene
    o = Oracle(threads=8)
    o.load_scene(s)
    info = o.gn_iteration(_params(s, forced_cg_iterations=1))      # the oracle fills in the column scale on a full iteration only
    r0 = o.rows(0)
    tw = np.array(list(info.type_weights))
    # E_g rows grouped like the engine's warps: the slot of a row is the rank of its voxel among the voxels with rows
    slot = np.unique(r0["voxel"], return_inverse=True)[1]
    eg = dict(voxel=r0["voxel"], frame=r0["aux"], residual=r0["residual"], raw_weight=r0["raw_weight"], J=o.eg_jacobian(),
              w_op=r0["weight"], slot=slot)
    R = ner.build_rows(s, eg, (o.rows(1), o.rows(2), o.rows(3)), tw)
    _, fm, cs = o.step()
    return R, fm.astype(bool), cs, info


def test_reference_reproduces_oracle_column_scale(oracle_rows):
    R, free, cs, info = oracle_rows
    assert R.eg["m"] == info.type_residuals[0] and free.sum() > 100
    out = ner.evaluate(R, free, np.zeros(R.U))
    s = out["s"][0]
    rel = np.abs(s[free] - cs[free]) / cs[free]
    assert rel.max() <= 1e-12, rel.max()
    assert np.all(s[~free] == 0.0)


def test_comparator_flags_small_errors(oracle_rows):
    R, free, _, _ = oracle_rows
    rng = np.random.default_rng(3)
    s_op = np.where(free, 0.5 + rng.random(R.U), 0.0)
    v = rng.standard_normal(R.U)
    counts = ner.rounding_counts(5)
    c = {k: counts["q" if k.startswith("q") else k] for k in ("s", "jtj", "b", "cam_acc", "q0")}
    base = ner.evaluate(R, free, s_op, [v])
    names = ("s", "jtj", "b", "cam_acc", "q0")
    # the exact values pass with ratio 0
    for k in names:
        assert ner.compare(base[k][0], base[k], c[k]) == (0.0, True, 0), k
    frame, slot = R.eg["frame"], R.eg["slot"]
    warp = np.nonzero(slot < 32)[0]
    f0 = np.bincount(frame[warp]).argmax()
    col = 2 * R.n + 6 * int(np.bincount(frame).argmax()) + 3
    cases = {
        "drop one E_g row": ner.Perturb(drop_eg_row=int(R.eg["m"] // 2)),
        "double one warp's pose contribution": ner.Perturb(pose_extra=(warp[frame[warp] == f0], 1.0)),
        "pose column scaled by 1 + 1e-5": ner.Perturb(col_scale=(col, 1.0 + 1e-5)),
    }
    for name, pert in cases.items():
        ref = ner.evaluate(R, free, s_op, [v], perturb=pert)
        flagged = [k for k in names if not ner.compare(base[k][0], ref[k], c[k])[1]]
        assert flagged, name
        print(name, "flagged by", flagged)
