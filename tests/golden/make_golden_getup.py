"""Fixture for HumanoidImGetup's reset: the UNMODIFIED reference's `_reset_actors`, `_reset_recovery_episode` and `_reset_fall_episode`
(phc/env/tasks/humanoid_im_getup.py:135-182), run on a stand-in task that carries the tensors they touch, over several reset rounds.

  * The stand-in subclasses the reference class without running its constructor (no simulator).  The reference-state branch,
    `super()._reset_actors(nonfall_ids)`, only records its env ids here: that part is pinned by the step / reset fixtures.
  * The reference's own draws come from the seeded torch RNG; `torch.bernoulli` and `torch.randperm` are wrapped to record their
    results, so the oracle can replay them in the injected form.
  * Case "a" has a pool of one fall state per env (the reference's layout) and runs enough rounds for stale assignments to be
    released (an env frees a state another env holds).  Case "b" has a smaller pool and runs until the reference's assertion
    (fewer free states than fall envs) fires; that round is recorded with the flag `assert`.
  * The attribute names the reference file uses are stored too (`names`, one space-separated string), so the test of the getup mixin's attribute contract needs no
    reference tree.

  python tests/golden/make_golden_getup.py     (needs the reference tree; writes tests/golden/getup.npz)
"""
import os
import re
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

CASES = {"a": dict(n=48, pool=48, rounds=10, p_rec=0.5, p_fall=0.4, steps=60, seed=11),
         "b": dict(n=48, pool=14, rounds=12, p_rec=0.2, p_fall=0.7, steps=150, seed=12)}


def main():
    from oracle.refshim.load_reference import REFERENCE_ROOT, load_reference
    load_reference()
    import importlib
    getup = importlib.import_module("phc.env.tasks.humanoid_im_getup")
    him = importlib.import_module("phc.env.tasks.humanoid_im")

    rec = {"bern": [], "perm": [], "ref": []}
    bern0, perm0 = torch.bernoulli, torch.randperm

    def bern(p, *a, **k):
        out = bern0(p, *a, **k)
        rec["bern"].append(out.clone())
        return out

    def perm(n, *a, **k):
        out = perm0(n, *a, **k)
        rec["perm"].append(out.clone())
        return out

    def ref_actors(self, env_ids):
        rec["ref"].append(env_ids.clone())

    torch.bernoulli, torch.randperm = bern, perm
    him.HumanoidIm._reset_actors = ref_actors            # what super()._reset_actors resolves to from HumanoidImGetup

    class Task(getup.HumanoidImGetup):
        def __init__(self):                              # no simulator: only the tensors _reset_actors touches
            pass

    out = {}
    for name, c in CASES.items():
        rng = np.random.default_rng(c["seed"])
        torch.manual_seed(c["seed"])
        n, pool = c["n"], c["pool"]
        t = Task()
        t.device = "cpu"
        t._recovery_episode_prob, t._fall_init_prob, t._recovery_steps = c["p_rec"], c["p_fall"], c["steps"]
        t.availalbe_fall_states = torch.zeros(pool, dtype=torch.long)
        t.fall_id_assignments = torch.zeros(n, dtype=torch.long)
        t._recovery_counter = torch.zeros(n, dtype=torch.int)
        t._humanoid_root_states = torch.from_numpy(rng.standard_normal((n, 13)).astype(np.float32))
        t._dof_pos = torch.from_numpy(rng.standard_normal((n, 69)).astype(np.float32))
        t._dof_vel = torch.from_numpy(rng.standard_normal((n, 69)).astype(np.float32))
        t._fall_root_states = torch.from_numpy(rng.standard_normal((pool, 13)).astype(np.float32))
        t._fall_dof_pos = torch.from_numpy(rng.standard_normal((pool, 69)).astype(np.float32))
        t._fall_dof_vel = torch.from_numpy(rng.standard_normal((pool, 69)).astype(np.float32))
        t._reset_fall_env_ids = []
        init = {"avail": t.availalbe_fall_states, "fid": t.fall_id_assignments, "rc": t._recovery_counter, "root": t._humanoid_root_states,
                "dof_pos": t._dof_pos, "dof_vel": t._dof_vel, "fall_root": t._fall_root_states, "fall_dof_pos": t._fall_dof_pos,
                "fall_dof_vel": t._fall_dof_vel}
        for k, v in init.items():
            out[f"{name}_init_{k}"] = v.numpy().copy()
        stale = 0
        r = 0
        for r in range(c["rounds"]):
            frac = [0.3, 0.6, 1.0][r % 3]
            env_ids = torch.from_numpy(np.flatnonzero(rng.random(n) < frac)).long()
            if env_ids.numel() == 0:
                env_ids = torch.tensor([0])
            t._terminate_buf = torch.from_numpy((rng.random(n) < 0.6).astype(np.int64))
            others = torch.ones(n, dtype=torch.bool)
            others[env_ids] = False
            held = t.fall_id_assignments[others]
            stale += int(sum(int(t.availalbe_fall_states[s]) == 1 and bool((held == s).any()) for s in t.fall_id_assignments[env_ids].tolist()))
            for v in rec.values():
                v.clear()
            p = f"{name}_r{r}_"
            out[p + "env_ids"], out[p + "terminate"] = env_ids.numpy(), t._terminate_buf.numpy().copy()
            asserted = 0
            try:
                t._reset_actors(env_ids)
            except AssertionError:
                asserted = 1
            out[p + "assert"] = np.array(asserted)
            out[p + "rec_bern"] = rec["bern"][0].numpy()
            out[p + "fall_bern"] = rec["bern"][1].numpy()
            out[p + "perm"] = rec["perm"][0].numpy() if rec["perm"] else np.zeros(0, np.int64)
            out[p + "ref_ids"] = rec["ref"][0].numpy() if rec["ref"] else np.zeros(0, np.int64)
            for k, v in (("avail", t.availalbe_fall_states), ("fid", t.fall_id_assignments), ("rc", t._recovery_counter),
                         ("root", t._humanoid_root_states), ("dof_pos", t._dof_pos), ("dof_vel", t._dof_vel)):
                out[p + k] = v.numpy().copy()
            if asserted:
                break
        out[f"{name}_rounds"] = np.array(r + 1)
        out[f"{name}_stale_releases"] = np.array(stale)
        for k in ("n", "pool", "p_rec", "p_fall", "steps"):
            out[f"{name}_{k}"] = np.array(c[k])
    torch.bernoulli, torch.randperm = bern0, perm0
    assert out["a_stale_releases"] > 0, "no stale release in case a: change the seed"
    assert out["b_r%d_assert" % (int(out["b_rounds"]) - 1)] == 1, "case b never exhausted its pool: change the seed"
    src = open(os.path.join(REFERENCE_ROOT, "phc", "env", "tasks", "humanoid_im_getup.py")).read()
    out["names"] = np.array(" ".join(sorted(set(re.findall(r"self\.([A-Za-z_][A-Za-z0-9_]*)", src)))))
    np.savez_compressed(os.path.join(HERE, "getup.npz"), **out)
    print("wrote getup.npz:", {k: int(out[f"{k}_rounds"]) for k in CASES}, "stale releases", int(out["a_stale_releases"]))


if __name__ == "__main__":
    main()
