"""The RGB-D renderer (k_render_fk + k_render, csrc/ge_render.cuh) pixel for pixel against the fp64 oracle's ray caster.

Both sides evaluate the same fp64 expressions on the same blob and break ties the same way (the lowest geom id wins), so every pixel's
f32 depth and u8 rgb must equal the oracle's, except where rounding can decide the answer.  The oracle's render probe
(OracleEnv.render_probe, orc_render_probe in oracle/grasp_oracle.c) names those pixels: silhouettes and hull edges that a ray moved by
EPS_PX pixels or an origin moved by EPS_M metres crosses, coplanar faces, u8 truncation and f32 rounding boundaries, checker lines.
The gate of every comparison: each mismatching pixel is flagged by the probe.  So that the probe cannot pass a test by flagging
everything, a fixed random sample of 2 000 pixels per image is probed too: over a test's images at most 0.1 % of the sampled pixels
may be flagged, and at most 0.5 % lie on a checker line.  The latter are real: the side camera looks horizontally, so the floor hits of
one image row share one depth, and near the horizon rows of far floor land exactly on checker lines in exact arithmetic (about 0.2 % of
its pixels; the oracle's own -ffp-contract=fast build renders 9-16 of them differently at 320 x 240).

EPS_PX = 1e-10 pixel and EPS_M = 1e-13 m: a ray direction that differs in its last bits (FMA contraction, 1e-16 relative) moves by about
1e-13 pixel, and geom frames that agree to 1e-15 m move a surface by about that much, so both are two to three orders of magnitude
above the differences the two sides can have, and ten orders below a pixel.  The f32-midpoint flag uses a relative 1e-12 window for the
same reason: at 1e-9 it would flag ~2 % of all pixels (the f32 spacing is 6e-8..1.2e-7 relative), with no rounding able to cross it.
Larger values flag too much where the depth is small: at EPS_M = 1e-12, 15 of the 2 000 sampled pixels of the top_down image with a
box face 1-30 mm from the camera were flagged.
The oracle's own -ffp-contract=fast build, which contracts to FMA as the GPU does, differs from the checker build on 434 pixels of 112
of these images; the probe flags all 434.

States: scene resets (scene B's unsettled, objects falling from 1.0-1.5 m next to the side camera at z = 1.0), the committed oracle
states of tests/golden/scene_a_edges.npz and scene_b_edges.npz, and objects placed by hand (rendering is kinematic, so interpenetration
does not matter): straddling each image border, a ball centred on a tile corner, a camera-aligned box whose silhouette lies on tile
boundaries (u = 31.5, v = 15.5 / 47.5: between pixel centres, so no pixel is decided by rounding), a ball 3 cm in front of the top_down
camera, a box straddling a camera's image plane (an OBB corner behind the camera: k_render_fk gives it the whole image) and one
entirely behind it.
"""
import os

import numpy as np
import pytest

from tests.common import reset_qpos_scene_a, reset_qpos_scene_b

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EPS_PX, EPS_M = 1e-10, 1e-13
SAMPLE, SAMPLE_RATE, SAMPLE_RATE_CHECKER = 2000, 1e-3, 5e-3
MAIN1, TOP_DOWN, SIDE = 0, 1, 2
SIZES = [(1, 1), (1, 200), (200, 1), (16, 16), (17, 15), (33, 31), (203, 77), (200, 200), (320, 240)]  # (W, H)
G_PLANE, G_SPHERE, G_CAPSULE, G_CYLINDER, G_BOX, G_MESH = 0, 2, 3, 5, 6, 7
RTILE = 16


# ------------------------------------------------------------------------------------------------ scenes and hand-placed states
_SCENES = {}


def _scene(S):
    """(blob, arrays, object geom ids by type, world offset of each object's free joint)"""
    if S not in _SCENES:
        from mujoco_rl_ur5_b200.model.scene import load_scene, load_scene_blob
        from oracle.oracle_py import OracleEnv

        A, _ = load_scene(S)
        blob = load_scene_blob(S)
        nq, ngeom = int(np.ravel(A["nq"])[0]), int(np.ravel(A["ngeom"])[0])
        nobj = (nq - 8) // 7
        gt = np.ravel(A["geom_type"])
        objs = {t: [g for g in range(ngeom - nobj, ngeom) if gt[g] == t] for t in (G_SPHERE, G_CAPSULE, G_CYLINDER, G_BOX)}
        q = _reset(S, A, 0)
        for i in range(nobj):
            q[8 + 7 * i:15 + 7 * i] = [0, 0, 0, 1, 0, 0, 0]
        o = OracleEnv(blob)
        o.reset(q)
        off = o.field("gpos").reshape(-1, 3)[ngeom - nobj:].copy()
        o.close()
        _SCENES[S] = (blob, A, objs, off, ngeom - nobj)
    return _SCENES[S]


def _reset(S, A, i):
    return (reset_qpos_scene_a if S == "A" else reset_qpos_scene_b)(A, i)


def _fixture(S):
    d = np.load(os.path.join(GOLDEN, "scene_a_edges.npz" if S == "A" else "scene_b_edges.npz"))
    return d["qpos"]


def _cam(A, cam, W, H):
    cp = np.asarray(A["cam_pos0"]).reshape(-1, 3)[cam]
    cm = np.asarray(A["cam_mat0"]).reshape(-1, 3, 3)[cam]
    f = 0.5 * H / np.tan(np.ravel(A["cam_fovy"])[cam] * np.pi / 360.0)
    return cp, cm, f


def _camera_point(A, cam, W, H, u, v, d):
    """camera-frame point seen at (fractional) pixel (u, v) at eye depth d: k_render_fk's pinhole c = W/2 - 1/2 - f x / (-z)"""
    _, _, f = _cam(A, cam, W, H)
    return np.array([(0.5 * W - 0.5 - u) * d / f, (0.5 * H - 0.5 - v) * d / f, -d])


def _quat(R):
    from scipy.spatial.transform import Rotation

    x, y, z, w = Rotation.from_matrix(R).as_quat()
    return np.array([w, x, y, z])


def _place(S, q, g, cam, W, H, p_cam, R_cam=None):
    """puts object geom g at camera-frame point p_cam of camera `cam`, its axes along R_cam (camera-frame columns; None: a fixed
    oblique orientation)"""
    blob, A, objs, off, first = _scene(S)
    cp, cm, _ = _cam(A, cam, W, H)
    if R_cam is None:
        from scipy.spatial.transform import Rotation

        R = Rotation.from_euler("xyz", [0.4, -0.7, 1.1]).as_matrix()
    else:
        R = cm @ R_cam
    a = 8 + 7 * (g - first)
    q[a:a + 3] = cp + cm @ p_cam - off[g - first]
    q[a + 3:a + 7] = _quat(R)


def _placed(S, cam, W, H):
    """objects straddling the four image borders, a ball centred on a tile corner, and a camera-aligned box whose silhouette lies on
    a tile column and a tile row boundary, all about 0.45 m in front of the camera"""
    blob, A, objs, off, first = _scene(S)
    q = _reset(S, A, 0)
    d = 0.45
    balls, boxes = objs[G_SPHERE], objs[G_BOX]
    caps = objs[G_CAPSULE] or balls[1:]
    cyls = objs[G_CYLINDER] or boxes[1:]
    _place(S, q, balls[0], cam, W, H, _camera_point(A, cam, W, H, -0.5, 0.3 * H, d))  # left border
    _place(S, q, boxes[0], cam, W, H, _camera_point(A, cam, W, H, W - 0.5, 0.6 * H, d))  # right border
    _place(S, q, caps[0], cam, W, H, _camera_point(A, cam, W, H, 0.4 * W, -0.5, d))  # top border
    _place(S, q, cyls[0], cam, W, H, _camera_point(A, cam, W, H, 0.7 * W, H - 0.5, d))  # bottom border
    _place(S, q, balls[-1], cam, W, H, _camera_point(A, cam, W, H, 15.5, 15.5, d))  # on the corner of four tiles
    # box face-on: its front face's +x edge (the silhouette while it lies right of the axis) on u = 31.5, its +y edge on v = 15.5/47.5
    g = boxes[-1]
    h = float(np.asarray(A["geom_size"]).reshape(-1, 3)[g, 0])
    u, v = (31.5 if W > 64 else 15.5), (47.5 if H > 96 else 15.5)
    e = _camera_point(A, cam, W, H, u, v, d - h)
    _place(S, q, g, cam, W, H, np.array([e[0] - h, e[1] - h, -d]), np.eye(3))
    return q


def _straddle(S, cam):
    """a camera-aligned box straddling the image plane (2 cm behind, 3 cm in front, its top face 1 mm below the camera: it fills most
    of the lower half of the image) and a box entirely behind the camera"""
    blob, A, objs, off, first = _scene(S)
    q = _reset(S, A, 0)
    boxes = objs[G_BOX]
    h = float(np.asarray(A["geom_size"]).reshape(-1, 3)[boxes[-1], 0])
    _place(S, q, boxes[-1], cam, 200, 200, np.array([0.0, -(h + 0.001), 0.02 - h]), np.eye(3))
    _place(S, q, boxes[0], cam, 200, 200, np.array([0.05, 0.0, 0.3]))
    return q


def _near(S):
    """the largest ball 3 cm in front of the top_down camera: it covers all but the image corners"""
    blob, A, objs, off, first = _scene(S)
    q = _reset(S, A, 0)
    sz = np.asarray(A["geom_size"]).reshape(-1, 3)
    g = max(objs[G_SPHERE], key=lambda g: sz[g, 0])
    _place(S, q, g, TOP_DOWN, 200, 200, np.array([0.0, 0.0, -(0.03 + sz[g, 0])]))
    return q


def _edge_cases(S):
    """(name, qpos, cam, W, H) of the culling-edge cases"""
    out = []
    for cam in (MAIN1, TOP_DOWN, SIDE):
        for W, H in ((200, 200), (203, 77)):
            out.append((f"{S} placed cam{cam} {W}x{H}", _placed(S, cam, W, H), cam, W, H))
            out.append((f"{S} straddle cam{cam} {W}x{H}", _straddle(S, cam), cam, W, H))
    out.append((f"{S} near top_down 200x200", _near(S), TOP_DOWN, 200, 200))
    out.append((f"{S} near top_down 203x77", _near(S), TOP_DOWN, 203, 77))
    return out


# ------------------------------------------------------------------------------------------------ k_render_fk's screen boxes, restated
def _screen_boxes(A, gpos, gmat, cam, W, H):
    """per geom: (raw box x0, y0, x1, y1 before clamping, clamped box, front); planes and geoms with an OBB corner less than 1e-6 in
    front of the camera get the whole image (front False), boxes off screen (1, 1, 0, 0)"""
    cp, cm, f = _cam(A, cam, W, H)
    gt = np.ravel(A["geom_type"])
    oc, oh = np.asarray(A["geom_obbcenter"]).reshape(-1, 3), np.asarray(A["geom_obbhalf"]).reshape(-1, 3)
    out = []
    for g in range(len(gt)):
        whole = (0, 0, W - 1, H - 1)
        if gt[g] == G_PLANE:
            out.append((None, whole, False))
            continue
        R = gmat[g].reshape(3, 3)
        t = gpos[g] + R @ oc[g] - cp
        us, vs, front = [], [], True
        for k in range(8):
            off = np.array([oh[g, 0] if k & 1 else -oh[g, 0], oh[g, 1] if k & 2 else -oh[g, 1], oh[g, 2] if k & 4 else -oh[g, 2]])
            qc = cm.T @ (R @ off + t)
            if -qc[2] < 1e-6:
                front = False
                break
            us.append(0.5 * W - 0.5 - f * qc[0] / -qc[2])
            vs.append(0.5 * H - 0.5 - f * qc[1] / -qc[2])
        if not front:
            out.append((None, whole, False))
            continue
        x0, x1 = int(np.floor(max(min(us), -2.0))) - 1, int(np.ceil(min(max(us), W + 1.0))) + 1
        y0, y1 = int(np.floor(max(min(vs), -2.0))) - 1, int(np.ceil(min(max(vs), H + 1.0))) + 1
        if x1 < 0 or x0 > W - 1 or y1 < 0 or y0 > H - 1:
            box = (1, 1, 0, 0)
        else:
            box = (max(x0, 0), max(y0, 0), min(x1, W - 1), min(y1, H - 1))
        out.append(((x0, y0, x1, y1), box, True))
    return out


def _largest_tile_list(boxes, W, H):
    b = np.array([bx[1] for bx in boxes])
    best = 0
    for r0 in range(0, H, RTILE):
        for c0 in range(0, W, RTILE):
            c1, r1 = min(W, c0 + RTILE), min(H, r0 + RTILE)
            meets = ~((b[:, 2] < c0) | (b[:, 0] > c1 - 1) | (b[:, 3] < r0) | (b[:, 1] > r1 - 1))
            best = max(best, int(meets.sum()))
    return best


def _oracle(S, qpos):
    from oracle.oracle_py import OracleEnv

    o = OracleEnv(_scene(S)[0])
    o.reset(qpos)
    return o


# ------------------------------------------------------------------------------------------------ CPU: what the cases reach
def test_render_cases_reach_the_culling_edges():
    """the hand-placed cases (with scene A's fixture states) show every geom type, clamp visible geoms at all four borders, put
    silhouettes on tile boundaries, show a geom with an OBB corner behind the camera, and leave background"""
    largest = {}
    for S in ("A", "B"):
        blob, A, objs, off, first = _scene(S)
        gt = np.ravel(A["geom_type"])
        cases = _edge_cases(S)
        if S == "A":
            cases += [(f"A fixture {i} cam{cam}", q, cam, 200, 200) for i, q in enumerate(_fixture("A")) for cam in (TOP_DOWN, SIDE)]
        type_px = {}
        clamped, tile_cols, tile_rows, behind, bg, offscreen = set(), 0, 0, 0, 0, 0
        for name, q, cam, W, H in cases:
            o = _oracle(S, q)
            gid, _ = o.render_probe(cam, W, H, eps_px=EPS_PX, eps_m=EPS_M)
            boxes = _screen_boxes(A, o.field("gpos").reshape(-1, 3), o.field("gmat").reshape(-1, 9), cam, W, H)
            o.close()
            seen = set(np.unique(gid[gid >= 0]).tolist())
            for g in seen:
                type_px[int(gt[g])] = type_px.get(int(gt[g]), 0) + int((gid == g).sum())
            for g in seen:
                raw, box, front = boxes[g]
                if raw is not None:
                    x0, y0, x1, y1 = raw
                    clamped |= {s for s, c in (("left", x0 < 0), ("top", y0 < 0), ("right", x1 > W - 1), ("bottom", y1 > H - 1)) if c}
                elif gt[g] != G_PLANE:
                    behind += 1
            offscreen += sum(1 for b in boxes if b[1] == (1, 1, 0, 0))
            bg += int((gid < 0).sum())
            for c in range(RTILE, W, RTILE):  # silhouettes between the last column of one tile and the first of the next
                tile_cols += int(((gid[:, c - 1] != gid[:, c]) & (np.maximum(gid[:, c - 1], gid[:, c]) >= first)).sum())
            for r in range(RTILE, H, RTILE):
                tile_rows += int(((gid[r - 1] != gid[r]) & (np.maximum(gid[r - 1], gid[r]) >= first)).sum())
            largest[name] = _largest_tile_list(boxes, W, H)
        want = [G_PLANE, G_SPHERE, G_BOX, G_MESH] + ([G_CAPSULE, G_CYLINDER] if S == "B" else [])
        print(f"scene {S}: pixels per geom type {type_px}, clamped at {sorted(clamped)}, object silhouettes on tile columns {tile_cols} "
              f"/ rows {tile_rows}, visible geoms with a corner behind the camera {behind}, background pixels {bg}, off-screen boxes "
              f"{offscreen}")
        assert all(type_px.get(t, 0) >= 20 for t in want), (S, type_px)
        assert clamped == {"left", "top", "right", "bottom"}, (S, clamped)
        assert tile_cols >= 20 and tile_rows >= 20, (S, tile_cols, tile_rows)
        assert behind >= 1 and bg > 0 and offscreen > 0, (S, behind, bg, offscreen)
    name = max(largest, key=largest.get)
    print(f"largest tile list: {largest[name]} geoms ({name})")
    assert largest[name] < 256


def test_render_probe_flags_rounding_decided_pixels_only():
    """the probe on scene A's top_down and side renders: interior pixels of a box face and of the floor are unflagged; with a ray
    moved by half a pixel every silhouette is flagged (of two neighbours seeing different geoms, at least one); at the chosen eps
    only a handful of pixels are flagged"""
    blob, A, objs, off, first = _scene("A")
    for cam, q in ((TOP_DOWN, _reset("A", A, 0)), (SIDE, _reset("A", A, 0)), (TOP_DOWN, _placed("A", TOP_DOWN, 200, 200))):
        o = _oracle("A", q)
        rgb, depth = o.render(cam, 200, 200)
        gid, fl = o.render_probe(cam, 200, 200, eps_px=EPS_PX, eps_m=EPS_M)
        # the probe picks orc_render's winner: background exactly where render() wrote the far plane with black
        assert np.array_equal(gid < 0, (depth == np.float32(50.0 * np.ravel(A["stat_extent"])[0])) & (rgb.max(axis=2) == 0))
        gt = np.ravel(A["geom_type"])
        same = np.ones_like(gid, bool)  # interior of a face: the 5 x 5 neighbourhood sees the same geom in the same colour
        for dr in range(-2, 3):
            for dc in range(-2, 3):
                same[2:-2, 2:-2] &= gid[2:-2, 2:-2] == gid[2 + dr:198 + dr, 2 + dc:198 + dc]
                same[2:-2, 2:-2] &= (rgb[2:-2, 2:-2] == rgb[2 + dr:198 + dr, 2 + dc:198 + dc]).all(axis=2)
        same[:2] = same[-2:] = False
        same[:, :2] = same[:, -2:] = False
        for t in (G_BOX, G_PLANE):
            inner = same & (gid >= 0) & (gt[np.maximum(gid, 0)] == t)
            if t == G_PLANE:  # off the checker lines: the checker colour changes there by design
                inner &= (fl & 16) == 0
            assert inner.sum() > (100 if t == G_BOX or cam == TOP_DOWN else -1), (cam, t)  # the side camera sees little near floor
            assert (fl[inner] & ~(4 | 8) == 0).all(), (cam, t, np.unique(fl[inner]))
            assert ((fl[inner] & (4 | 8)) != 0).sum() <= 1e-3 * inner.sum()
        _, wide = o.render_probe(cam, 200, 200, eps_px=0.5, eps_m=EPS_M)
        for a, b in ((np.s_[:, :-1], np.s_[:, 1:]), (np.s_[:-1, :], np.s_[1:, :])):
            edge = gid[a] != gid[b]
            assert edge.sum() > 50
            assert (((wide[a] & 1) != 0) | ((wide[b] & 1) != 0))[edge].all(), (cam, int(edge.sum()))
        n = int((fl != 0).sum())
        print(f"cam {cam}: {n} of 40000 pixels flagged at eps_px {EPS_PX}, eps_m {EPS_M}; {int((wide != 0).sum())} at eps_px 0.5")
        assert n <= 100, n
        o.close()


# ------------------------------------------------------------------------------------------------ GPU comparisons
def _render(S, states, cam, W, H, engine=None):
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    eng = engine or BatchedEngine(_scene(S)[0], len(states), 0)
    eng.set_state(np.stack(states))
    rgb, depth = eng.render(cam, W, H)
    out = rgb.cpu().numpy(), depth.cpu().numpy()
    if engine is None:
        eng.close()
    return out


class Gate:
    """every mismatching pixel flagged by the probe; counts per image and a pooled sample flag rate"""

    def __init__(self):
        self.rows, self.failures = [], []

    def check(self, S, q, cam, W, H, rgb, depth, what):
        o = _oracle(S, q)
        orgb, odepth = o.render(cam, W, H)
        diff = (depth.view(np.uint32) != odepth.view(np.uint32)) | (rgb != orgb).any(axis=2)
        idx = np.flatnonzero(diff)
        fl = o.render_probe(cam, W, H, idx, EPS_PX, EPS_M)[1] if len(idx) else np.zeros(0, np.int32)
        # the sample leaves out the central column / row of an odd width / height: its rays have an exact 0 in the camera frame, so they
        # lie in the scene's symmetry plane x = 0 (top_down) or are exactly horizontal (side), and every one of them is flagged
        r, c = np.divmod(np.arange(W * H), W)
        pool = np.flatnonzero(~((W % 2 == 1) & (c == W // 2)) & ~((H % 2 == 1) & (r == H // 2)))
        sample = np.random.RandomState(W * 7919 + H * 31 + cam).choice(pool, min(SAMPLE, len(pool)), replace=False)
        sfl = o.render_probe(cam, W, H, sample, EPS_PX, EPS_M)[1]
        o.close()
        self.rows.append((what, len(idx), int((fl != 0).sum()), int(((sfl != 0) & (sfl & 16 == 0)).sum()), int((sfl & 16 != 0).sum()),
                          len(sample)))
        bad = idx[fl == 0]
        if len(bad):
            p = bad[:4]
            self.failures.append(f"{what}: {len(bad)} unflagged mismatches, e.g. (row, col) {[(int(i // W), int(i % W)) for i in p]} "
                                 f"depth {depth.ravel()[p].tolist()} vs {odepth.ravel()[p].tolist()}, rgb {rgb.reshape(-1, 3)[p].tolist()} "
                                 f"vs {orgb.reshape(-1, 3)[p].tolist()}")

    def finish(self):
        mism = sum(r[1] for r in self.rows)
        flagged = sum(r[2] for r in self.rows)
        sf, sc, sn = (sum(r[k] for r in self.rows) for k in (3, 4, 5))
        for r in self.rows:
            if r[1] or r[3] or r[4]:
                print(f"  {r[0]}: {r[1]} mismatching pixels ({r[2]} flagged); of {r[5]} sampled pixels {r[3]} flagged, {r[4]} on checker lines")
        print(f"{len(self.rows)} images: {mism} mismatching pixels, {flagged} of them flagged; sampled pixels flagged {sf} / {sn}, "
              f"on checker lines {sc} / {sn}")
        assert not self.failures, "\n".join(self.failures)
        assert sf <= SAMPLE_RATE * sn and sc <= SAMPLE_RATE_CHECKER * sn, (sf, sc, sn)


def _gpu_states_a():
    blob, A, objs, off, first = _scene("A")
    return [_reset("A", A, 0), _reset("A", A, 1)] + list(_fixture("A"))


@pytest.mark.gpu
def test_cameras_and_sizes_scene_a():
    """scene A (warp-per-env build): all three cameras at every size of SIZES (square, single row / column, below one tile,
    non-square both ways), and the side camera at 1000 x 1000 (the picture of GraspEnv's recorded grasps)"""
    gate = Gate()
    base = _gpu_states_a()
    for cam in (MAIN1, TOP_DOWN, SIDE):
        for W, H in SIZES + ([(1000, 1000)] if cam == SIDE else []):
            states = base + [_placed("A", cam, W, H)]
            rgb, depth = _render("A", states, cam, W, H)
            for i, q in enumerate(states):
                gate.check("A", q, cam, W, H, rgb[i], depth[i], f"A cam{cam} {W}x{H} state {i}")
    gate.finish()


@pytest.mark.gpu
def test_scene_b_edge_states_and_unsettled_resets():
    """scene B (CTA-per-env build): the 12 edge states and four unsettled resets, top_down 200 x 200, side 320 x 240, main1 203 x 77"""
    blob, A, objs, off, first = _scene("B")
    states = list(_fixture("B")) + [_reset("B", A, i) for i in range(4)]
    gate = Gate()
    for cam, W, H in ((TOP_DOWN, 200, 200), (SIDE, 320, 240), (MAIN1, 203, 77)):
        rgb, depth = _render("B", states, cam, W, H)
        for i, q in enumerate(states):
            gate.check("B", q, cam, W, H, rgb[i], depth[i], f"B cam{cam} {W}x{H} state {i}")
    gate.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("S", ["A", "B"])
def test_culling_edges(S):
    """the hand-placed cases: geoms clamped at the borders, silhouettes on tile boundaries, a corner behind the camera (whole-image
    box), geoms behind the camera, off-screen boxes, a ball covering most tiles"""
    gate = Gate()
    groups = {}
    for name, q, cam, W, H in _edge_cases(S):
        groups.setdefault((cam, W, H), []).append((name, q))
    for (cam, W, H), cases in groups.items():
        rgb, depth = _render(S, [q for _, q in cases], cam, W, H)
        for i, (name, q) in enumerate(cases):
            gate.check(S, q, cam, W, H, rgb[i], depth[i], name)
    gate.finish()


def _batch_states(n):
    blob, A, objs, off, first = _scene("A")
    states = [_reset("A", A, i) for i in range(n)]
    special = {0: _placed("A", SIDE, 400, 480), 1: _straddle("A", SIDE), n - 1: _placed("A", TOP_DOWN, 200, 200), n // 2: _near("A")}
    for k, q in zip((2, n // 2 - 1, n - 2, 3000, 3729), _fixture("A")):
        special[k] = q
    for k, q in special.items():
        states[k] = q
    return states, sorted(special) + [17, 1234]


@pytest.mark.gpu
def test_4096_envs_each_render_what_one_env_renders():
    """4096 distinct scene-A states: each image equals the same state rendered by a 1-env engine, bit for bit, at top_down 200 x 200
    and at side 400 x 480, where the rgb byte offsets pass 2^31 from env 3729 on (2.4 GB rgb + 3.1 GB depth)"""
    import torch

    from mujoco_rl_ur5_b200.engine import BatchedEngine

    n = 4096
    states, check = _batch_states(n)
    eng = BatchedEngine(_scene("A")[0], n, 0)
    one = BatchedEngine(_scene("A")[0], 1, 0)
    eng.set_state(np.stack(states))
    for cam, W, H in ((TOP_DOWN, 200, 200), (SIDE, 400, 480)):
        rgb, depth = eng.render(cam, W, H)
        if W == 400:
            assert 3 * n * W * H > 2 ** 31 and 3 * 3729 * W * H > 2 ** 31
        for k in check:
            one.set_state(states[k][None])
            r1, d1 = one.render(cam, W, H)
            assert torch.equal(rgb[k], r1[0]) and torch.equal(depth[k].view(torch.int32), d1[0].view(torch.int32)), (cam, W, H, k)
        gate = Gate()
        for k in (0, n - 1):
            gate.check("A", states[k], cam, W, H, rgb[k].cpu().numpy(), depth[k].cpu().numpy(), f"batch env {k} cam{cam} {W}x{H}")
        gate.finish()
        del rgb, depth
        torch.cuda.empty_cache()
    eng.close()
    one.close()


@pytest.mark.gpu
def test_a_large_render_between_two_small_ones_changes_nothing():
    """top_down 200 x 200, then side 1000 x 1000, then top_down 200 x 200 again on one engine: the last image equals the first"""
    import torch

    from mujoco_rl_ur5_b200.engine import BatchedEngine

    states = _gpu_states_a()[:4]
    eng = BatchedEngine(_scene("A")[0], len(states), 0)
    eng.set_state(np.stack(states))
    r1, d1 = [t.clone() for t in eng.render(TOP_DOWN, 200, 200)]
    eng.render(SIDE, 1000, 1000)
    r2, d2 = eng.render(TOP_DOWN, 200, 200)
    assert torch.equal(r1, r2) and torch.equal(d1.view(torch.int32), d2.view(torch.int32))
    eng.close()


def _engine(S, n, **env):
    from mujoco_rl_ur5_b200.engine import BatchedEngine

    for k, v in env.items():
        os.environ[k] = str(v)
    try:
        return BatchedEngine(_scene(S)[0], n, 0)
    finally:
        for k in env:
            del os.environ[k]


def _outputs(eng, q, v):
    """render, debug_forward, step_open_loop and body_xpos of one engine on the states (q, v)"""
    eng.set_state(q, v)
    rgb, depth = eng.render(TOP_DOWN, 200, 200)
    out = {"rgb": rgb.cpu().numpy(), "depth": depth.cpu().numpy(), "xpos": eng.body_xpos().cpu().numpy()}
    for f in ("qacc", "contact", "qfrc_constraint"):
        out[f] = np.concatenate([eng.debug_forward(e, f) for e in range(len(q))])
    eng.step_open_loop(5)
    out["qpos_after"] = eng.get_state()[0].cpu().numpy()
    return out


@pytest.mark.gpu
def test_two_engines_with_different_workspaces_live_side_by_side():
    """scene A at GE_MAXCON 512 and 256 (workspaces above 48 KB of different sizes; the opt-in to them is per kernel, not per
    engine): created in both orders and used in both orders, every output equals what a fresh engine alone gives"""
    d = np.load(os.path.join(GOLDEN, "scene_a_edges.npz"))
    q, v = d["qpos"][:2], d["qvel"][:2]
    alone, size = {}, {}
    for mc in (512, 256):
        e = _engine("A", 2, GE_MAXCON=mc)
        size[mc] = e.size(7)
        alone[mc] = _outputs(e, q, v)
        e.close()
    print(f"workspace bytes per env: GE_MAXCON 512 {size[512]}, 256 {size[256]}")
    assert size[512] > size[256] > 48 * 1024
    for first, second in ((512, 256), (256, 512)):
        for use in ((first, second), (second, first)):
            engines = {first: _engine("A", 2, GE_MAXCON=first)}
            engines[second] = _engine("A", 2, GE_MAXCON=second)
            for mc in use:
                got = _outputs(engines[mc], q, v)
                for k, x in alone[mc].items():
                    assert x.shape == got[k].shape and np.array_equal(x, got[k]), (first, second, use, mc, k)
            for e in engines.values():
                e.close()


@pytest.mark.gpu
def test_render_and_pixel_2_world_reject_bad_arguments():
    """GE_ERR_ARG for a camera outside [0, ncam) and for a width or height above 32767 (16-bit screen boxes); GE_ERR_MODEL for a
    scene with more geoms than the renderer's 256-entry tile list"""
    import ctypes as C

    import torch

    from mujoco_rl_ur5_b200.engine import BatchedEngine
    from mujoco_rl_ur5_b200.model import blob as blobmod

    GE_ERR_ARG, GE_ERR_MODEL = -1, -3
    eng = BatchedEngine(_scene("A")[0], 1, 0)
    L, h = eng.L, eng.h
    rgb = torch.zeros(32768 * 3, dtype=torch.uint8, device="cuda")
    depth = torch.zeros(32768, dtype=torch.float32, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    for cam in (-1, 3, 1 << 20):
        assert L.ge_render(h, cam, 16, 16, p(rgb), p(depth)) == GE_ERR_ARG, cam
    assert L.ge_render(h, TOP_DOWN, 32768, 1, p(rgb), p(depth)) == GE_ERR_ARG
    assert L.ge_render(h, TOP_DOWN, 1, 32768, p(rgb), p(depth)) == GE_ERR_ARG
    assert L.ge_render(h, TOP_DOWN, 16, 16, p(rgb), p(depth)) == 0
    px = torch.zeros(1, dtype=torch.int32, device="cuda")
    d1 = torch.ones(1, dtype=torch.float32, device="cuda")
    xyz = torch.zeros(3, dtype=torch.float64, device="cuda")
    for cam in (-1, 3):
        assert L.ge_pixel_2_world(h, cam, 200, 200, p(px), p(px), p(d1), p(xyz)) == GE_ERR_ARG, cam
    assert L.ge_pixel_2_world(h, TOP_DOWN, 200, 200, p(px), p(px), p(d1), p(xyz)) == 0
    torch.cuda.synchronize()
    eng.close()
    arrays = blobmod.unpack(_scene("A")[0])
    arrays["ngeom"] = np.array([257], np.int32)
    hh = C.c_void_p()
    blob = blobmod.pack(arrays)
    assert L.ge_create(blob, len(blob), 1, 0, None, C.byref(hh)) == GE_ERR_MODEL
