"""The info dict of FurnitureEnv.step over the CPU envs of oracle/ref_env.py (TEST INFRASTRUCTURE): _compute_reward's four terms
(furniture.py:482-550), FurnitureBaxterEnv's "ac" (furniture_baxter.py:75) and _after_step's episode record (:451-480).

with_step_info(cls) gives a CPU env class whose step() also leaves `step_info`, the info dict the reference's step returns, with its keys
in the reference's order.  The reward is restated with its terms, in the arithmetic of OracleFurnitureEnv._compute_reward; the episode's
return is summed from each step's reward before the penalty, and a reset zeroes it (_after_reset, :351-362), the reset inside an unstable
step included (_do_simulation's except branch, :2889-2897)."""
import time
from collections import OrderedDict

import numpy as np

TERMS = ("success_reward", "touch_reward", "pick_reward", "ctrl_penalty")
EPISODE = ("episode_success", "episode_reward", "episode_length", "episode_time", "episode_unstable", "episode_num_connected")


class StepInfoMixin:
    def reset(self):
        ob = super().reset()
        self.episode_reward, self.episode_time = 0.0, time.time()
        return ob

    def _compute_reward(self, raw, fail):  # FurnitureEnv._compute_reward with its info (furniture.py:482-541)
        touch_r = pick_r = 0.0
        if not fail:
            bits = self.touch_bits()
            for arm in range(self.narms):
                both = 3 if arm == 0 else 24
                for p in range(self.npart):
                    if bits[p] & both == both:
                        if not self.touched[p]:
                            self.touched[p] = True; touch_r += self.cfg.touch_reward
                        if not (bits[p] & 4) and not self.picked[p]:
                            self.picked[p] = True; pick_r += self.cfg.pick_reward
        success_r = self.cfg.success_reward * (self.num_connected - self.prev_num_connected)
        self.prev_num_connected = self.num_connected
        ctrl = -self.cfg.ctrl_penalty_coef * float(np.square(raw).sum())  # _ctrl_penalty (:543-550)
        reward = success_r + touch_r + pick_r + ctrl
        self.terms = OrderedDict(zip(TERMS, (success_r, touch_r, pick_r, ctrl)))
        self.episode_reward += reward  # _after_step (:459-461)
        success = self.num_connected == getattr(self, "success_num_conn", self.npart - 1) and self.npart > 1
        return reward, success, success

    def step(self, action):
        ob, reward, done, info = super().step(action)
        penalty = -float(self.cfg.unstable_penalty_coef) if info["unstable"] else 0
        d = OrderedDict(self.terms)
        if self.narms == 2:  # FurnitureBaxterEnv._step (furniture_baxter.py:75)
            d["ac"] = np.asarray(action)
        if done:  # _after_step (:469-478)
            vals = (int(info["success"]), self.episode_reward + penalty, self.episode_len, time.time() - self.episode_time, penalty, self.num_connected)
            d.update(zip(EPISODE, vals))
            if info["success"]:
                d["episode_success_state"] = {"qpos": np.array(self.sim.qpos), "qvel": np.array(self.sim.qvel)}
        self.step_info = d
        return ob, reward, done, info


def with_step_info(cls):
    """cls (a CPU env of oracle/ with the sparse reward) with the step's info dict: instances leave it in `step_info` after every step"""
    return type("StepInfo" + cls.__name__, (StepInfoMixin, cls), {})
