"""Shared helpers for the parity tests: drive the engine (CUDA build on the GPU box, lane-emulated harness on CPU)
and the CPU oracle from the same state and compare stage by stage."""
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU_DIR = os.path.join(ROOT, "tests", "emu")
EMU_LIB = os.path.join(EMU_DIR, "libfe_emu.so")


def build_emu():
    src = os.path.join(EMU_DIR, "fe_emu.cpp")
    csrc = os.path.join(ROOT, "furniture_b200", "csrc")
    deps = [src, os.path.join(ROOT, "include", "furniture_b200.h")] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".h", ".inl"))]
    if not os.path.exists(EMU_LIB) or any(os.path.getmtime(d) > os.path.getmtime(EMU_LIB) for d in deps):
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-w", "-o", EMU_LIB, src])
    return EMU_LIB


def have_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def make_engine(model, n_envs, use_gpu, **cfg):
    from furniture_b200.engine import Engine, default_config

    c = default_config(**cfg)
    if use_gpu:
        return Engine(model, n_envs, device=0, config=c)
    return Engine(model, n_envs, config=c, lib_path=build_emu())


def joint_qadr(model, names):
    """qpos addresses of the named (hinge / slide) joints"""
    return np.array([model.jnt_qposadr[model.names["jnt"].index(n)] for n in names], dtype=np.int64)


def arm_qadr(model):
    """qpos addresses of the agent's arm joints and of its gripper joints, in the order of robot_init_qpos /
    gripper_init_qpos (Baxter: the head pan is dof 0 and every arm has its gripper after it, so neither set is contiguous)"""
    return joint_qadr(model, model.meta["robot_joints"]), joint_qadr(model, model.meta["gripper_joints"])


def settled_state(model, seed=0, robot_noise=0.3, dz=0.01):
    """qpos with parts at their XML init poses (+dz) and the arm near its init pose."""
    rng = np.random.RandomState(seed)
    q = model.qpos0.copy()
    meta = model.meta
    arm, grip = arm_qadr(model)
    q[arm] = meta["robot_init_qpos"] + rng.uniform(-robot_noise, robot_noise, len(arm))
    q[grip] = meta["gripper_init_qpos"]
    for name in meta["part_names"]:
        qa = model.jnt_qposadr[model.names["jnt"].index(name)]
        if name in meta["part_init_qpos"]:
            q[qa : qa + 7] = meta["part_init_qpos"][name]  # else: the XML body pose (already in qpos0)
        q[qa + 2] += dz
    return q


def to_z(model, em, xmat_links, qacc):
    """oracle qacc (MuJoCo dof order: v, w_local per part) -> engine solver coordinates [alpha_world; vdot]."""
    z = np.array(qacc, dtype=np.float64).copy()
    nr = em.nrlink
    for p in range(em.npart):
        R = xmat_links[nr + p].reshape(3, 3)
        da = nr + 6 * p
        z[da : da + 3] = R @ qacc[da + 3 : da + 6]
        z[da + 3 : da + 6] = qacc[da : da + 3]
    return z


def oracle_link_poses(sim, em):
    xpos = sim.xpos.reshape(-1, 3)
    xquat = sim.xquat.reshape(-1, 4)
    xmat = sim.xmat.reshape(-1, 9)
    idx = em.link_body
    return xpos[idx], xquat[idx], xmat[idx]


def quat_err(a, b):
    return min(np.abs(a - b).max(), np.abs(a + b).max())
