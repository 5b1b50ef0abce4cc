"""FurnitureCursorEnv (BASELINE.json config 1: Cursor + toy_table, 1 env) over the C-ABI simulator surface.

The Cursor agent has no robot: two box "cursors" (static bodies moved through ``sim.model.body_pos``, margin = size, gap = 10:
contacts that are reported but never push, robots/cursor/robot.xml:4-7) select furniture parts, carry them around and ask for
connections.  Its logic is a sequence of small host-side decisions with a ``sim.forward(); sim.step()`` between most of them
(`_move_rotate_object` -> `_is_inside`, furniture.py:771-783), so it is written here as host code over the simulator entry
points (fe_sim_forward / fe_sim_step / fe_get_field / fe_set_field / fe_is_aligned), mirroring the reference method by method:

  _step_discrete            furniture/env/furniture.py:800-845        move / rotate / select per cursor, connect request
  _move_cursor              :712-727                                  boundary test, position through the model
  _move_rotate_object       :729-757                                  rigid move of the selected group, rolled back if it leaves the box
  _is_inside, _get_bounding_box  :749-783
  _select_object, on_collision   :785-798, :3290-3310                 cursor contacts (sensor geoms: touch flags of the engine)
  _try_connect (10-step slerp / lerp approach, then _connect)         :926-1042
  _connect, _align_connectors, _activate_weld                         :847-924, :1224-1250, :2761-2776
  _do_simulation (Cursor branch: gravity compensation of the selected groups)  :2857-2897
  _reset (Cursor branches) and UniformRandomSampler                   :1406-1663, models/tasks/placement_sampler.py:137-190
  _get_obs                  furniture.py:1344-1387, furniture_cursor.py:98-116
  _compute_reward / _after_step   furniture.py:482-541, :451-480

The simulator behind it is pluggable (``backend``): the engine (``EngineBackend``: the CUDA library with one env, or the
lane-emulated build in the CPU tests) or any object with the same handful of methods (the tests drive the fp64 oracle through
the same logic to check decisions and poses).
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np

from . import mjcf
from .mjcf import q_conj, q_mul, q_to_mat


# ---- pyquaternion / transform_utils semantics the reference's geometry goes through (float64; transform_utils.py:617-664)
def _qinv(q):
    q = np.asarray(q, dtype=np.float64)
    return np.array([q[0], -q[1], -q[2], -q[3]]) / float(q @ q)


def _qrot(q, v):
    q = np.asarray(q, dtype=np.float64)
    n = math.sqrt(float(q @ q))
    if abs(1.0 - n) >= 1e-14 and n > 0:  # Quaternion.rotate normalises first
        q = q / n
    return q_mul(q_mul(q, np.array([0.0, v[0], v[1], v[2]])), q_conj(q))[1:]


def euler_to_quat(rotation, quat=None):
    """T.euler_to_quat: extrinsic x, y, z rotations in degrees, applied after `quat` (transform_utils.py:617-630)"""
    def ax(axis, deg):
        h = math.radians(deg) / 2
        return np.array([math.cos(h)] + [math.sin(h) * a for a in axis])

    q = q_mul(q_mul(ax([0, 0, 1], rotation[2]), ax([0, 1, 0], rotation[1])), ax([1, 0, 0], rotation[0]))
    return q if quat is None else q_mul(np.asarray(quat, dtype=np.float64), q)


def rel_pose(qpos1, qpos2):
    inv = _qinv(qpos1[3:])
    return np.concatenate([_qrot(inv, np.asarray(qpos2[:3]) - np.asarray(qpos1[:3])), q_mul(inv, np.asarray(qpos2[3:], dtype=np.float64))])


def transform_to_target_quat(qpos_base, qpos, target_quat):
    """pose of `qpos` after its base is turned from its own quaternion to `target_quat` about the base position (:641-664)"""
    rel = q_mul(np.asarray(target_quat, dtype=np.float64), _qinv(qpos_base[3:]))
    new_pos = _qrot(rel, np.asarray(qpos[:3]) - np.asarray(qpos_base[:3])) + np.asarray(qpos_base[:3])
    return new_pos, q_mul(rel, np.asarray(qpos[3:], dtype=np.float64))


def _unit_vector_f32(v):  # transform_utils.unit_vector as it is in force: float32 copy (the second definition wins, :559-590)
    d = np.array(v, dtype=np.float32, copy=True)
    d /= math.sqrt(np.dot(d, d))
    return d


def quat_slerp(quat0, quat1, fraction):
    """T.quat_slerp (transform_utils.py:122-159), shortest path, no spin"""
    q0, q1 = _unit_vector_f32(quat0[:4]), _unit_vector_f32(quat1[:4])
    if fraction == 0.0:
        return q0
    if fraction == 1.0:
        return q1
    d = np.dot(q0, q1)
    if abs(abs(d) - 1.0) < np.finfo(float).eps * 4.0:
        return q0
    if d < 0.0:
        d = -d
        q1 *= -1.0
    d = min(d, 1.0)
    angle = math.acos(d)
    if abs(angle) < np.finfo(float).eps * 4.0:
        return q0
    isin = 1.0 / math.sin(angle)
    q0 *= math.sin((1.0 - fraction) * angle) * isin
    q1 *= math.sin(fraction * angle) * isin
    q0 += q1
    return q0


class EngineBackend:
    """the handful of MjSim operations the cursor logic needs, on one env of the engine (C-ABI: fe_sim_forward, fe_sim_step,
    fe_get_field / fe_set_field, fe_is_aligned)"""

    def __init__(self, model, device=0, lib_path=None):
        from .engine import Engine, default_config

        self.model = model
        self.eng = Engine(model, 1, device=device, config=default_config(), lib_path=lib_path)
        self.em = self.eng.em
        self._cursor_model = self.eng.get("static_pos")[0].reshape(2, 3).astype(np.float64)
        self._cursor_data = self._cursor_model.copy()
        self._contype0, self._conaff0 = self.eng.get("geom_contype")[0].copy(), self.eng.get("geom_conaffinity")[0].copy()

    def reset_data(self):  # MjSim.reset(): data only
        m = self.model
        self.eng.set("qpos", m.qpos0); self.eng.set("qvel", np.zeros(m.nv)); self.eng.set("qacc_warmstart", np.zeros(m.nv))
        self.eng.set("gravcomp", np.zeros(self.em.npart))

    def forward(self):
        self.eng.set("static_pos", self._cursor_model.reshape(1, 6))
        self.eng.forward()
        self._cursor_data = self._cursor_model.copy()

    def step(self, n=1):
        self.eng.set("static_pos", self._cursor_model.reshape(1, 6))
        self.eng.step(n)
        self._cursor_data = self._cursor_model.copy()

    def qpos(self):
        return self.eng.get("qpos")[0].astype(np.float64)

    def set_qpos(self, q):
        self.eng.set("qpos", np.asarray(q, dtype=np.float32))

    def qvel(self):
        return self.eng.get("qvel")[0].astype(np.float64)

    def set_qvel(self, v):
        self.eng.set("qvel", np.asarray(v, dtype=np.float32))

    def zero_warmstart(self):
        self.eng.set("qacc_warmstart", np.zeros(self.model.nv))

    def set_gravcomp(self, factors):  # xfrc_applied = -factor * gravity * mass at the CoM of every part (furniture.py:2778-2790)
        self.eng.set("gravcomp", np.asarray(factors, dtype=np.float32))

    def part_poses(self):  # (npart, 3), (npart, 4) of the last forward / step
        nrl = self.em.nrlink
        return self.eng.get("link_xpos")[0].reshape(-1, 3)[nrl:].astype(np.float64), self.eng.get("link_xquat")[0].reshape(-1, 4)[nrl:].astype(np.float64)

    def cursor_pos(self, i):  # data xpos: what the last forward / step saw
        return self._cursor_data[i].copy()

    def set_cursor_pos(self, i, pos):  # sim.model.body_pos[...] = pos
        self._cursor_model[i] = np.asarray(pos, dtype=np.float64)

    def touch_bits(self):  # per part: bit 0 cursor0, bit 1 cursor1 touch one of its geoms (sensor contacts of the last forward / step)
        return self.eng.get("touch")[0]

    def geom_masks(self):
        return self.eng.get("geom_contype")[0].copy(), self.eng.get("geom_conaffinity")[0].copy()

    def set_geom_masks(self, ct, ca):
        self.eng.set("geom_contype", ct); self.eng.set("geom_conaffinity", ca)

    def engine_geom(self, model_geom):  # model geom id -> index in the engine's (colliding-only) geom tables, or None
        return self.em.geom_map.get(model_geom)

    def eq(self):
        return self.eng.get("eq_active")[0].copy(), self.eng.get("eq_data")[0].reshape(-1, 7).copy()

    def set_eq(self, active, data):
        self.eng.set("eq_active", active); self.eng.set("eq_data", np.asarray(data, dtype=np.float32).reshape(1, -1))

    def is_aligned(self, p1, m1, p2, m2, angles, thr):
        ang = np.zeros((1, 4)); ang[0, : len(angles)] = angles
        ok, tq = self.eng.is_aligned([p1], [np.ravel(m1)], [p2], [np.ravel(m2)], ang, [len(angles)], [list(thr)])
        return bool(ok[0]), (None if np.isnan(tq[0]).any() else tq[0])

    def close(self):
        self.eng.close()


class FurnitureCursorEnvB200:
    def __init__(self, furniture_name="toy_table", backend=None, device=0, lib_path=None, seed=123, move_speed=0.1, rotate_speed=22.5,
                 cursor_boundary=1.5, max_episode_steps=100, furn_xyz_rand=0.02, furn_rot_rand=3.0, success_reward=100.0, auto_align=True,
                 alignment_pos_dist=0.1, alignment_rot_dist_up=0.9, alignment_rot_dist_forward=0.9, alignment_project_dist=0.3, control_freq=10,
                 furniture_id=None, **ignored):
        """`furniture_id` and the remaining keywords (id, name, background, port ...) are what gym passes from the registration
        (env/__init__.py:19-34: IKEACursor-v0, furniture_id 0); renderer options are ignored"""
        if furniture_id is not None and furniture_name == "toy_table" and "furniture_name" not in ignored:
            from .env import FURNITURE_NAMES

            furniture_name = FURNITURE_NAMES[int(furniture_id)]
        if ignored.get("no_collision"):
            raise ValueError("no_collision is built for the robot envs, not the Cursor env")
        if ignored.get("assembled"):
            raise ValueError("assembled is built for the robot envs, not the Cursor env")
        self.ignored_config = sorted(ignored)
        self.model = m = backend.model if backend is not None else mjcf.load_scene("Cursor", furniture_name)
        self.sim = backend if backend is not None else EngineBackend(m, device=device, lib_path=lib_path)
        self.cfg = dict(move_speed=move_speed, rotate_speed=rotate_speed, cursor_boundary=cursor_boundary, max_episode_steps=max_episode_steps,
                        furn_xyz_rand=furn_xyz_rand, furn_rot_rand=furn_rot_rand, success_reward=success_reward, auto_align=auto_align)
        self.thr = (alignment_pos_dist, alignment_rot_dist_up, alignment_rot_dist_forward, alignment_project_dist)
        self.parts = list(m.meta["part_names"])
        self.npart = len(self.parts)
        self.part_body = [m.names["body"].index(n) for n in self.parts]
        self.part_qadr = [int(m.jnt_qposadr[m.names["jnt"].index(n)]) for n in self.parts]
        self.part_dadr = [int(m.jnt_dofadr[m.names["jnt"].index(n)]) for n in self.parts]
        self.conn_sites = [s for s, n in enumerate(m.names["site"]) if "conn_site" in n]
        self.part_sites = [[s for s in range(m.nsite) if m.site_bodyid[s] == b] for b in self.part_body]
        self.cursor_geoms = [m.names["geom"].index("cursor0"), m.names["geom"].index("cursor1")]
        self.part_col_geoms = [g for g, n in enumerate(m.names["geom"]) if "collision" in n and m.names["body"][m.geom_bodyid[g]] in self.parts]
        self.nsub = int((1.0 / control_freq) / m.opt_timestep)
        self.rng = np.random.RandomState(seed)
        self.dof = 15  # (move 3, rotate 3, select 1) x 2 + connect (furniture_cursor.py:52-58)
        self.num_connect_steps = 10
        self._gravcomp = np.zeros(self.npart)

    # ---- small helpers (furniture.py names in the comments)
    def _find(self, i):  # _find_group
        while self.group[i] != i:
            i = self.group[i]
        return i

    def _q(self, p):  # _get_qpos
        return self.sim.qpos()[self.part_qadr[p] : self.part_qadr[p] + 7]

    def _set_q(self, p, pos, quat):  # _set_qpos
        q = self.sim.qpos()
        q[self.part_qadr[p] : self.part_qadr[p] + 3] = pos
        q[self.part_qadr[p] + 3 : self.part_qadr[p] + 7] = quat
        self.sim.set_qpos(q)

    def _stop(self, parts, gravity):  # _stop_object: gravity-compensation factor, zero velocity
        v = self.sim.qvel()
        for p in parts:
            self._gravcomp[p] = gravity
            v[self.part_dadr[p] : self.part_dadr[p] + 6] = 0
        self.sim.set_qvel(v)
        self.sim.set_gravcomp(self._gravcomp)

    def _slow(self):  # _slow_objects
        v = self.sim.qvel()
        for p in range(self.npart):
            self._gravcomp[p] = 1.0
            v[self.part_dadr[p] : self.part_dadr[p] + 6] = np.clip(v[self.part_dadr[p] : self.part_dadr[p] + 6], -0.2, 0.2)
        self.sim.set_qvel(v)
        self.sim.set_gravcomp(self._gravcomp)

    def _fwd_step(self):
        self.sim.forward()
        self.sim.step()

    def _site_pose(self, s, xpos, xquat):
        m = self.model
        p = self.part_body.index(int(m.site_bodyid[s]))
        R = q_to_mat(xquat[p])
        return xpos[p] + R @ m.site_pos[s], R @ q_to_mat(m.site_quat[s]), q_mul(xquat[p], m.site_quat[s])

    def _selected_groups(self):
        return [self._find(p) for p in self.cursor_selected if p is not None]

    # ---- reset (furniture.py:1406-1663, Cursor branches)
    def _place(self):
        """UniformRandomSampler.sample (placement_sampler.py:137-190), draw for draw"""
        m, placed, out = self.model, [], []
        xy, rot_r = self.cfg["furn_xyz_rand"], self.cfg["furn_rot_rand"]
        for name in self.parts:
            init, r = m.meta["part_init_qpos"][name], m.meta["part_radius"][name]
            for _ in range(10000):
                x = init[0] + self.rng.uniform(-xy, xy)
                y = init[1] + self.rng.uniform(-xy, xy)
                if all(np.linalg.norm([x - px, y - py], 2) > pr + r for px, py, pr in placed):
                    break
            rot = self.rng.uniform(high=rot_r, low=rot_r)
            placed.append((x, y, r))
            out.append((np.array([x, y, init[2] + 0.01]), euler_to_quat([rot, 0, 0], init[3:7])))
        return out

    def _init_cursors(self):  # _initialize_robot_pos, :1777-1779
        h = self.cfg["move_speed"] / 2
        self.sim.set_cursor_pos(0, [-0.2, 0.0, h])
        self.sim.set_cursor_pos(1, [0.2, 0.0, h])

    def reset(self):
        sim, m = self.sim, self.model
        sim.reset_data()
        ct, ca = sim.geom_masks()
        saved = {}
        for g in self.cursor_geoms:  # robot collision off during the furniture settle phase (:1441-1453)
            e = sim.engine_geom(g)
            saved[e] = (ct[e], ca[e])
            ct[e] = ca[e] = 0
        for g in self.part_col_geoms:
            e = sim.engine_geom(g)
            ct[e] = ca[e] = 1
        sim.set_geom_masks(ct, ca)
        self.group = list(range(self.npart))
        self.connected_sites, self.num_connected, self.prev_num_connected = set(), 0, 0
        self.cursor_selected, self.connect_step, self.connected_body1 = [None, None], 0, None
        act, data = sim.eq()
        act[:] = 0
        sim.set_eq(act, data)
        self._gravcomp[:] = 0
        for p, (pos, quat) in enumerate(self._place()):
            self._set_q(p, pos, quat)
        for _ in range(10):  # stabilise furniture (:1535-1540)
            self._stop(range(self.npart), 0)
            for _ in range(10):
                self._fwd_step()
                self._slow()
        self._init_cursors()
        self._fwd_step()
        ct, ca = sim.geom_masks()
        for e, (a, b) in saved.items():
            ct[e], ca[e] = a, b
        sim.set_geom_masks(ct, ca)
        for _ in range(100):
            self._init_cursors()
            self._fwd_step()
        self._gravcomp[:] = 0  # sync (:1621-1628): xfrc_applied = 0, warm start cleared
        sim.set_gravcomp(self._gravcomp)
        sim.zero_warmstart()
        sim.forward()
        for _ in range(100):
            self._fwd_step()
        self.episode_len, self.episode_reward, self.success = 0, 0.0, False
        return self._obs()

    # ---- step pieces
    def _move_cursor(self, i, offset):  # :712-727
        pos = self.sim.cursor_pos(i) + offset
        b = self.cfg["cursor_boundary"]
        if (np.abs(pos) < b).all() and pos[2] >= self.cfg["move_speed"] * 0.45:
            self.sim.set_cursor_pos(i, pos)
            return True
        return False

    def _bounding_min_max(self, obj):  # _get_bounding_box :749-769 (both start from 0)
        xpos, xquat = self.sim.part_poses()
        g = self._find(obj)
        mn, mx = np.zeros(3), np.zeros(3)
        for p in range(self.npart):
            if self._find(p) == g:
                for s in self.part_sites[p]:
                    sp = self._site_pose(s, xpos, xquat)[0]
                    mn, mx = np.minimum(mn, sp), np.maximum(mx, sp)
        return mn, mx

    def _is_inside(self, obj):  # :771-783
        self._fwd_step()
        mn, mx = self._bounding_min_max(obj)
        b = self.cfg["cursor_boundary"]
        return not ((mn < np.array([-b, -b, -0.05])).any() or (mx > np.array([b, b, b])).any())

    def _move_rotate_object(self, obj, move_offset, rotate_offset):  # :729-747
        base = self._q(obj)
        target_quat = euler_to_quat(rotate_offset, base[3:])
        g, old = self._find(obj), {}
        for p in range(self.npart):
            if self._find(p) == g:
                old[p] = self._q(p)
                npos, nq = transform_to_target_quat(base, old[p], target_quat)
                self._set_q(p, npos + move_offset, nq)
        if self._is_inside(obj):
            return True
        for p, q in old.items():
            self._set_q(p, q[:3], q[3:])
        return False

    def _select_object(self, i):  # :785-798
        bits = self.sim.touch_bits()
        for p in range(self.npart):
            if self._find(p) in self._selected_groups():
                continue
            if bits[p] & (1 << i):
                return p
        return None

    def _move_group_to(self, obj, target_pos, target_quat, gravity):  # _move_objects_target :1155-1176
        base = self._q(obj)
        translation = np.asarray(target_pos) - base[:3]
        g = self._find(obj)
        for p in range(self.npart):
            if self._find(p) == g:
                npos, nq = transform_to_target_quat(base, self._q(p), target_quat)
                self._set_q(p, npos + translation, nq)
                self._stop([p], gravity)

    def _try_connect(self, part1, part2):  # :926-1042
        m = self.model
        g1, g2 = self._find(part1), self._find(part2)
        sites1 = [s for s in self.conn_sites if self._find(self.part_body.index(int(m.site_bodyid[s]))) == g1]
        sites2 = [s for s in self.conn_sites if self._find(self.part_body.index(int(m.site_bodyid[s]))) == g2]
        if not sites1 or not sites2:
            return False
        bodies = [self.part_body[p] for p in range(self.npart) if self._find(p) in (g1, g2)]
        if not any(int(a) in bodies and int(b) in bodies for a, b in zip(m.eq_obj1id, m.eq_obj2id)):
            return False
        xpos, xquat = self.sim.part_poses()
        for s1 in sites1:
            n1 = m.names["site"][s1]
            for s2 in sites2:
                if s1 in self.connected_sites or s2 in self.connected_sites:
                    continue
                n2 = m.names["site"][s2]
                if n1.split(",")[0].split("-") != n2.split(",")[0].split("-")[::-1]:
                    continue
                p1, m1, q1 = self._site_pose(s1, xpos, xquat)
                p2, m2, q2 = self._site_pose(s2, xpos, xquat)
                angles = [float(x) for x in n1.split(",")[1:-1] if x]
                ok, tq = self.sim.is_aligned(p1, m1, p2, m2, angles, self.thr)
                if tq is not None:
                    self.target_quat = tq
                if not ok:
                    continue
                if self.connect_step < self.num_connect_steps:  # approach: 10 interpolated poses, one per connect action
                    body2 = self.part_body.index(int(m.site_bodyid[s2]))
                    part2_q = self._q(body2)
                    site2_pose = np.concatenate([p2, q2])
                    body_pos, body_rot = transform_to_target_quat(site2_pose, part2_q, self.target_quat)
                    body_pos = body_pos + (p1 - p2)
                    if self.connect_step == 0:
                        n = self.num_connect_steps
                        self.next_rot = [quat_slerp(part2_q[3:], body_rot, (f + 1) * 1 / n) for f in range(n)]
                        xnew = np.linspace(1 / n, 0.9, n)  # interp1d over [0, 1] between the two positions (:1016-1024)
                        self.next_pos = [part2_q[:3] + x * (body_pos - part2_q[:3]) for x in xnew]
                    self._move_group_to(body2, self.next_pos[self.connect_step], [float(v) for v in self.next_rot[self.connect_step]], 1)
                    self.connect_step += 1
                    return False
                self._connect(s1, s2, p1, q1, p2, q2)
                self.connect_step = 0
                self.next_pos = self.next_rot = None
                return True
        self.connect_step = 0
        return False

    def _connect(self, s1, s2, p1, q1, p2, q2):  # :847-924
        m, sim = self.model, self.sim
        self.connected_sites |= {s1, s2}
        body1, body2 = self.part_body.index(int(m.site_bodyid[s1])), self.part_body.index(int(m.site_bodyid[s2]))
        g1, g2 = self._find(body1), self._find(body2)
        ct, ca = sim.geom_masks()
        for g in range(m.ngeom):
            b = int(m.geom_bodyid[g])
            e = sim.engine_geom(g)
            if e is not None and b in self.part_body and self._find(self.part_body.index(b)) in (g1, g2) and ct[e] != 0:
                ct[e], ca[e] = (1 << 30) - 1 - (1 << (g1 + 1)), 1 << (g1 + 1)
        sim.set_geom_masks(ct, ca)
        if self.cfg["auto_align"]:  # _align_connectors / _move_site_to_target (:1224-1250), gravity = _gravity_compensation = 1
            base, bq = np.concatenate([p2, q2]), self._q(body2)
            _, nq = transform_to_target_quat(base, bq, self.target_quat)
            nsp, _ = transform_to_target_quat(bq, base, nq)
            tr = p1 - nsp
            g = self._find(body2)
            qb = self._q(body2)
            for p in range(self.npart):
                if self._find(p) == g:
                    npos, nqq = transform_to_target_quat(qb, self._q(p), nq)
                    self._set_q(p, npos + tr, nqq)
                    self._stop([p], 1)
        self._stop([p for p in range(self.npart) if self._find(p) in self._selected_groups()], 1)  # _stop_selected_objects
        self._fwd_step()
        mn = np.minimum(self._bounding_min_max(body1)[0], self._bounding_min_max(body2)[0])
        if mn[2] < 0:
            off = np.array([0, 0, -mn[2]])
            self._move_rotate_object(body1, off, [0, 0, 0])
            self._move_rotate_object(body2, off, [0, 0, 0])
        self._stop([p for p in range(self.npart) if self._find(p) in self._selected_groups()], 1)
        self._fwd_step()
        act, data = sim.eq()
        for e in range(m.neq):  # _activate_weld :2761-2776
            a, b = self.part_body.index(int(m.eq_obj1id[e])), self.part_body.index(int(m.eq_obj2id[e]))
            if a in (body1, body2) and b in (body1, body2):
                data[e] = rel_pose(self._q(a), self._q(b))
                act[e] = 1
                self.group[self._find(body1)] = self._find(body2)
        sim.set_eq(act, data)
        self.cursor_selected[1] = None  # release cursor
        self.num_connected += 1
        self.connected_body1, self.connected_pose = body1, self._q(body1)

    def _step_discrete(self, a):  # :800-845
        acts = [a[:7], a[7:14]]
        for i in range(2):
            move, rot, select = acts[i][0:3] * self.cfg["move_speed"], acts[i][3:6] * self.cfg["rotate_speed"], acts[i][6] > 0
            if not select:
                self.cursor_selected[i] = None
            if not self._move_cursor(i, move):
                continue
            if self.cursor_selected[i] is not None:
                if not self._move_rotate_object(self.cursor_selected[i], move, rot):
                    self._move_cursor(i, -move)
                    continue
            if select and self.cursor_selected[i] is None:
                self.cursor_selected[i] = self._select_object(i)
        if a[14] > 0 and self.cursor_selected[0] is not None and self.cursor_selected[1] is not None:
            self._try_connect(self.cursor_selected[0], self.cursor_selected[1])
        elif self.connect_step > 0:
            self.connect_step = 0

    def _obs(self):  # furniture.py:1344-1387 + furniture_cursor.py:98-116
        xpos, xquat = self.sim.part_poses()
        ob = OrderedDict()
        ob["object_ob"] = np.concatenate([np.concatenate([xpos[p], xquat[p]]) for p in range(self.npart)])
        ob["robot_ob"] = np.concatenate([self.sim.cursor_pos(0), self.sim.cursor_pos(1),
                                         [float(self.cursor_selected[0] is not None), float(self.cursor_selected[1] is not None)]])
        return ob

    def step(self, action):
        a = np.asarray(action["default"] if isinstance(action, dict) else action, dtype=np.float64).copy()
        assert a.shape == (15,)
        self._step_discrete(a)
        # _do_simulation(None), Cursor branch (:2865-2886): selected groups float, the others get their velocity zeroed
        sel = self._selected_groups()
        for p in range(self.npart):
            self._stop([p], 1 if self._find(p) in sel else 0)
        self.sim.forward()
        self.sim.step(self.nsub)
        self._stop([p for p in range(self.npart) if self._find(p) in sel], 1)
        if self.connected_body1 is not None:  # :426-436
            self.sim.forward()
            self._move_group_to(self.connected_body1, self.connected_pose[:3], self.connected_pose[3:], 1)
            self.connected_body1 = None
            self._fwd_step()
        ob = self._obs()
        done = self.num_connected == self.npart - 1 and self.npart > 1
        self.success = self.success or done
        reward = self.cfg["success_reward"] * (self.num_connected - self.prev_num_connected)  # no touch / pick / control terms for the Cursor (:489, :547)
        self.prev_num_connected = self.num_connected
        self.episode_reward += reward
        self.episode_len += 1
        info = {}
        if self.episode_len == self.cfg["max_episode_steps"]:
            done = True
        if done:
            info = dict(episode_success=int(self.success), episode_reward=self.episode_reward, episode_length=self.episode_len, episode_unstable=0,
                        episode_num_connected=self.num_connected)
        return ob, reward, done, info

    def get_env_state(self):  # :1781-1792
        return {"qpos": self.sim.qpos(), "qvel": self.sim.qvel(), "cursor0": self.sim.cursor_pos(0), "cursor1": self.sim.cursor_pos(1)}

    def close(self):
        if hasattr(self.sim, "close"):
            self.sim.close()
