"""CPU oracle of HumanoidImGetup's reset (TEST INFRASTRUCTURE): `_reset_actors` / `_reset_recovery_episode` / `_reset_fall_episode`
(phc/env/tasks/humanoid_im_getup.py:135-182) restated with injected draws, composed with `oracle.pulse_oracle.reset_envs` for the
reference-state subset.  Pinned to the unmodified reference by tests/golden/getup.npz (make_golden_getup.py).

Injected draws, the form `pulse_reset_getup` consumes: per env a recovery and a fall uniform (a Bernoulli draw succeeds when u < p),
per fall state a non-negative key (the free states in ascending (key, state id) order are the reference's randperm of them).
`draws_from_reference` turns the reference's recorded Bernoulli results and permutation into that form."""
from typing import Dict, Optional, Tuple

import torch

from oracle import pulse_oracle as po

REF, FALL, RECOVERY = 1, 2, 3


def draws_from_reference(env_ids: torch.Tensor, terminate_buf: torch.Tensor, avail: torch.Tensor, fid: torch.Tensor, rec_bern: torch.Tensor,
                         fall_bern: torch.Tensor, perm: Optional[torch.Tensor], num_envs: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(recovery_u [N], fall_u [N], fall_keys [P]) reproducing the reference's draws for one `_reset_actors(env_ids)` call:
    `rec_bern` over env_ids, `fall_bern` over the non-recovery envs, `perm` the randperm over the free states (None: no fall env).
    A success becomes u = 0 (< p whenever p > 0, the only case it can occur), a failure u = 1 (never < p <= 1); the free state at
    position perm[i] of the ascending free list gets key i."""
    rec_u, fall_u = torch.ones(num_envs), torch.ones(num_envs)
    rec_u[env_ids] = torch.where(rec_bern == 1, 0.0, 1.0)
    rec = (rec_bern == 1) & (terminate_buf[env_ids] == 1)
    fall_u[env_ids[~rec]] = torch.where(fall_bern == 1, 0.0, 1.0)
    keys = torch.zeros(avail.shape[0])
    if perm is not None and perm.numel() > 0:
        free = _released(avail, fid, env_ids).eq(0).nonzero().flatten()
        keys[free[perm]] = torch.arange(perm.numel(), dtype=torch.float32)
    return rec_u, fall_u, keys


def _released(avail, fid, env_ids):
    a = avail.clone()
    a[fid[env_ids]] = 0
    return a


def getup_reset_actors(st: Dict[str, torch.Tensor], env_ids: torch.Tensor, recovery_u: torch.Tensor, fall_u: torch.Tensor,
                       fall_keys: torch.Tensor, recovery_prob: float, fall_prob: float, recovery_steps: int):
    """`_reset_actors(env_ids)` without its reference-state part.  st keys: terminate_buf, recovery_counter (int32), avail, fid (int64),
    root_states [N,13], dof_pos / dof_vel [N,69], fall_root [P,13], fall_dof_pos / fall_dof_vel [P,69].  Returns (updated copies,
    info) with info: ref_ids / fall_ids / recovery_ids (ascending), fall_states (state of each fall env), classes [N] (0 = not reset)
    and shortfall.  Where the reference asserts (more fall envs than free states, :172) the surplus fall envs, the last ones in env
    order, take a reference-state episode and `shortfall` counts them."""
    o = {k: v.clone() for k, v in st.items()}
    ids = env_ids.long()
    o["avail"][o["fid"][ids]] = 0                                    # :136, stale assignments included
    rec = (recovery_u[ids] < recovery_prob) & (o["terminate_buf"][ids] == 1)
    rec_ids = ids[rec]
    o["recovery_counter"][rec_ids] = recovery_steps                  # _reset_recovery_episode
    non = ids[~rec]
    fall_ids = non[fall_u[non] < fall_prob]
    free = o["avail"].eq(0).nonzero().flatten()
    order = free[torch.argsort(fall_keys[free], stable=True)]        # ascending key, ties in state order
    take = min(fall_ids.numel(), free.numel())
    surplus = fall_ids[take:]
    fall_ids, states = fall_ids[:take], order[:take]
    o["root_states"][fall_ids] = o["fall_root"][states]              # _reset_fall_episode
    o["dof_pos"][fall_ids] = o["fall_dof_pos"][states]
    o["dof_vel"][fall_ids] = o["fall_dof_vel"][states]
    o["recovery_counter"][fall_ids] = recovery_steps
    o["avail"][states] = 1
    o["fid"][fall_ids] = states
    ref_ids = torch.sort(torch.cat([non[fall_u[non] >= fall_prob], surplus])).values
    o["recovery_counter"][ref_ids] = 0
    classes = torch.zeros(o["terminate_buf"].shape[0], dtype=torch.uint8)
    classes[ref_ids], classes[fall_ids], classes[rec_ids] = REF, FALL, RECOVERY
    return o, {"ref_ids": ref_ids, "fall_ids": fall_ids, "recovery_ids": rec_ids, "fall_states": states, "classes": classes,
               "shortfall": int(surplus.numel())}


def getup_reset(tb, cfg, st: Dict[str, torch.Tensor], env_ids: torch.Tensor, phase: torch.Tensor, recovery_u: torch.Tensor,
                fall_u: torch.Tensor, fall_keys: torch.Tensor, recovery_prob: float, fall_prob: float, recovery_steps: int,
                num_amp_steps: int = 10):
    """The whole device-side reset: `getup_reset_actors`, `po.reset_envs` on the reference-state envs (start-time draw, MotionLib
    state, AMP back-fill, their counters), then `_reset_env_tensors` (humanoid.py:603-606) on every reset env.  `st` also carries the
    keys `po.reset_envs` reads."""
    o, info = getup_reset_actors(st, env_ids, recovery_u, fall_u, fall_keys, recovery_prob, fall_prob, recovery_steps)
    o = po.reset_envs(tb, cfg, o, info["ref_ids"], phase, num_amp_steps)
    ids = env_ids.long()
    for k in ("progress_buf", "reset_buf", "terminate_buf", "contact_forces"):
        o[k][ids] = 0
    return o, info


def getup_amp_init(amp_obs_buf: torch.Tensor, body_state: torch.Tensor, dof_pos: torch.Tensor, dof_vel: torch.Tensor, fall_ids: torch.Tensor,
                   recovery_ids: torch.Tensor) -> torch.Tensor:
    """`_init_amp_obs` for the fall and recovery envs after the refresh (humanoid_amp.py:519-533, humanoid_im_getup.py:190-196): row 0 <-
    the current AMP observation (`_compute_amp_observations(env_ids)`), and for fall envs every history row too
    (`_init_amp_obs_default`).  body_state [N,24,13]."""
    out = amp_obs_buf.clone()
    ids = torch.cat([fall_ids, recovery_ids]).long()
    if ids.numel() == 0:
        return out
    bs = body_state[ids]
    cur = po.amp_obs_smpl(bs[:, 0, 0:3], bs[:, 0, 3:7], bs[:, 0, 7:10], bs[:, 0, 10:13], dof_pos[ids], dof_vel[ids],
                          bs[:, list(po.KEY_BODY_IDS), 0:3], po.amp_dof_subset())
    out[ids, 0] = cur
    nf = fall_ids.numel()
    out[fall_ids.long(), 1:] = cur[:nf, None]
    return out
