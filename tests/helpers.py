"""Shared test helpers: golden-fixture loading and oracle table construction (test infra)."""
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def load_npz(name):
    with np.load(os.path.join(GOLDEN, name)) as z:
        return {k: torch.from_numpy(z[k]) if z[k].ndim > 0 else z[k].item() for k in z.files}


def oracle_tables(device="cpu"):
    from oracle.pulse_oracle import MotionTables
    z = load_npz("motionlib.npz")
    return MotionTables(**{k: v.to(device) for k, v in z.items()})


def clip_rates(fps, num_motions):
    """Per-clip frame rates as float64 [M]: a scalar for every clip, or a sequence repeated over the clips in order."""
    r = torch.tensor(fps if isinstance(fps, (list, tuple)) else [fps], dtype=torch.float64)
    return r.repeat((num_motions + r.numel() - 1) // r.numel())[:num_motions]


def synthetic_tables(num_motions, seed=0, min_frames=5, max_frames=400, median_frames=150, fps=30.0):
    """AMASS-shaped flat MotionLib tables written directly (SURVEY 8d): unit quaternions, smooth
    positions; bypasses the reference's 60 ms/clip loader.  Returns oracle MotionTables on CPU.
    fps: one rate, or a sequence of per-clip rates (clip_rates); length and dt follow the reference's
    `1.0 / fps * (num_frames - 1)` and `1.0 / fps` in float64, stored as float32 (motion_lib_base.py:262-263)."""
    from oracle.pulse_oracle import MotionTables
    rng = np.random.default_rng(seed)
    nf = np.clip(np.exp(rng.normal(np.log(median_frames), 0.6, size=num_motions)).astype(np.int64), min_frames, max_frames)
    F = int(nf.sum())
    g = torch.Generator().manual_seed(seed)

    def unit(x):
        return torch.nn.functional.normalize(x, dim=-1)

    base_q = unit(torch.randn(num_motions, 24, 4, generator=g)).repeat_interleave(torch.from_numpy(nf), dim=0)
    grs = unit(base_q + 0.15 * torch.randn(F, 24, 4, generator=g))
    lrs = unit(torch.randn(num_motions, 24, 4, generator=g).repeat_interleave(torch.from_numpy(nf), dim=0)
               + 0.15 * torch.randn(F, 24, 4, generator=g))
    base_p = (torch.randn(num_motions, 24, 3, generator=g) * 0.4 + torch.tensor([0.0, 0.0, 0.9])).repeat_interleave(torch.from_numpy(nf), dim=0)
    gts = base_p + 0.05 * torch.randn(F, 24, 3, generator=g)
    gvs = torch.randn(F, 24, 3, generator=g)
    gavs = torch.randn(F, 24, 3, generator=g)
    dvs = torch.randn(F, 23, 3, generator=g)
    aa = torch.randn(F, 72, generator=g)
    nf_t = torch.from_numpy(nf)
    starts = torch.cumsum(nf_t, 0) - nf_t
    rates = clip_rates(fps, num_motions).tolist()
    lengths = torch.tensor([(1.0 / r) * (int(n) - 1) for r, n in zip(rates, nf)], dtype=torch.float32)
    dt = torch.tensor([1.0 / r for r in rates], dtype=torch.float32)
    return MotionTables(gts=gts, grs=grs, lrs=lrs, gvs=gvs, gavs=gavs, dvs=dvs, motion_aa=aa, lengths=lengths,
                        num_frames=nf_t, dt=dt, length_starts=starts, fps=torch.tensor(rates, dtype=torch.float32),
                        motion_bodies=torch.zeros(num_motions, 17), motion_limb_weights=torch.zeros(num_motions, 10))


def synthetic_step_inputs(tb, n_envs, seed=0, dt=None):
    """Per-env task buffers + simulator state near the reference pose (SURVEY 8d), on CPU."""
    from oracle import pulse_oracle as po
    dt = po.STEP_DT if dt is None else dt
    g = torch.Generator().manual_seed(seed + 1)
    M = tb.num_motions
    motion_ids = torch.arange(n_envs) % M
    L = tb.lengths[motion_ids]
    progress = torch.randint(0, 40, (n_envs,), generator=g)
    start = po.sample_time_interval(tb, motion_ids, torch.rand(n_envs, generator=g))
    start_off = torch.zeros(n_envs)
    goff = torch.zeros(n_envs, 3)
    goff[::4, :2] = torch.randn((n_envs + 3) // 4, 2, generator=g)
    cycle = torch.zeros(n_envs, dtype=torch.int32)
    cycle[::7] = 5
    t = po.im_motion_times(progress, start, start_off, dt, plus_one=False)
    pose = po.motion_state(tb, motion_ids, t, goff)
    noise = torch.full((n_envs, 1, 1), 0.03)
    noise[::5] = 0.12
    body_pos = pose["rg_pos"] + noise * torch.randn(n_envs, 24, 3, generator=g)
    dq = torch.nn.functional.normalize(torch.cat([0.1 * torch.randn(n_envs, 24, 3, generator=g), torch.ones(n_envs, 24, 1)], -1), dim=-1)
    body_rot = torch.nn.functional.normalize(po.quat_mul(pose["rb_rot"], dq), dim=-1)
    body_vel = pose["body_vel"] + 0.5 * torch.randn(n_envs, 24, 3, generator=g)
    body_ang = pose["body_ang_vel"] + 0.5 * torch.randn(n_envs, 24, 3, generator=g)
    return {
        "motion_ids": motion_ids, "progress_buf": progress, "start_times": start, "start_offset": start_off,
        "global_offset": goff, "cycle_counter": cycle,
        "body_state": torch.cat([body_pos, body_rot, body_vel, body_ang], dim=-1).contiguous(),
        "dof_pos": pose["dof_pos"] + 0.05 * torch.randn(n_envs, 69, generator=g),
        "dof_vel": pose["dof_vel"] + 0.5 * torch.randn(n_envs, 69, generator=g),
        "dof_force": 30 * torch.randn(n_envs, 69, generator=g),
        "reset_buf_in": torch.zeros(n_envs, dtype=torch.long),
    }


def vae_golden():
    """tests/golden/vae.npz (reference-generated, make_golden_vae.py) + the oracle's view of its network weights."""
    from oracle import pulse_oracle as po
    g = load_npz("vae.npz")
    S, Tk, A, E, T, NE = [int(x) for x in g["dims"]]
    sd = {k[4:]: v for k, v in g.items() if k.startswith("net.")}
    nets = po.VaeNets.from_state_dict(sd, S)
    pnn_cols = [([g[f"pnn.actors.{c}.{i}.weight"] for i in (0, 2, 4)], [g[f"pnn.actors.{c}.{i}.bias"] for i in (0, 2, 4)]) for c in range(3)]
    composer = ([g[f"composer.{i}.weight"] for i in (0, 2, 4)], [g[f"composer.{i}.bias"] for i in (0, 2, 4)])
    return g, sd, nets, dict(S=S, Tk=Tk, A=A, E=E, T=T, NE=NE), pnn_cols, composer


def vae_param_list(nets):
    """Trainable tensors of the kin loss in reference naming order -> {reference parameter name: tensor}."""
    out = {}
    for name, (ws, bs) in (("z_mlp", nets.enc), ("z_prior", nets.prior), ("actor_mlp", (nets.dec[0][:-1], nets.dec[1][:-1]))):
        for i, (w, b) in enumerate(zip(ws, bs)):
            out[f"{name}.{2 * i}.weight"], out[f"{name}.{2 * i}.bias"] = w, b
    for name, (w, b) in (("z_mu", nets.enc_mu), ("z_logvar", nets.enc_logvar), ("z_prior_mu", nets.prior_mu),
                         ("z_prior_logvar", nets.prior_logvar), ("mu", (nets.dec[0][-1], nets.dec[1][-1]))):
        out[f"{name}.weight"], out[f"{name}.bias"] = w, b
    return out


# ----------------------------------------------------------------------------------------------------------------------
# Full-width (im_z_fit.yaml) PULSE VAE fixture: 16 M parameters cannot be committed, so weights and inputs are REGENERATED
# from integer draws (torch.randint on a seeded CPU generator: exact integers, identical on every host) by the SAME
# function in the golden generator (tests/golden/make_golden_vae_full.py) and in the tests; the fixture stores a float64
# checksum of what was generated plus the reference's outputs.
# ----------------------------------------------------------------------------------------------------------------------
VAE_FULL = dict(S=358, Tk=576, A=69, E=32, T=32, NE=64, task_units=(1536, 1024, 512), dec_units=(3096, 2048, 1024))


def _uniform_pm1(shape, gen):
    """exact: integers in [0, 2^16) -> (-1, 1) on a 2^-15 grid"""
    return (torch.randint(0, 65536, shape, generator=gen).float() - 32767.5) * (1.0 / 32768.0)


def _approx_normal(shape, gen):
    """sum of four uniforms, unit variance (exact arithmetic on small integers)"""
    s = torch.randint(0, 65536, (4,) + tuple(shape), generator=gen).sum(0).float()
    return (s - 2.0 * 65535.0) * (1.0 / (65536.0 * (4.0 / 12.0) ** 0.5))


def vae_full_fixture(seed=2024):
    """state dict (reference parameter names, no prefix) + minibatch of the im_z_fit.yaml-sized PULSE VAE.
    Weight scale: U(-1/sqrt(K), 1/sqrt(K)) like nn.Linear's default; biases small but non-zero."""
    d = VAE_FULL
    S, Tk, A, E, T, NE = d["S"], d["Tk"], d["A"], d["E"], d["T"], d["NE"]
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def lin(name, n_out, n_in, wscale=1.0, bscale=0.05):
        sd[name + ".weight"] = _uniform_pm1((n_out, n_in), g) * (wscale / n_in ** 0.5)
        sd[name + ".bias"] = _uniform_pm1((n_out,), g) * bscale

    def stack(name, n_in, units):
        for i, u in enumerate(units):
            lin(f"{name}.{2 * i}", u, n_in, wscale=2.0)    # gain that keeps the SiLU stacks' activations O(1)
            n_in = u
        return n_in

    tu, du = list(d["task_units"]), list(d["dec_units"])
    n = stack("z_mlp", S + Tk, tu + [5 * E])
    lin("z_mu", E, n)
    lin("z_logvar", E, n, wscale=3.0, bscale=1.0)          # a spread of log-variances, some past the [-5, 2] clamp
    n = stack("z_prior", S, tu)
    lin("z_prior_mu", E, n)
    lin("z_prior_logvar", E, n, wscale=3.0, bscale=1.0)
    n = stack("actor_mlp", S + E, du)
    lin("mu", A, n)
    B = T * NE
    obs = torch.clamp(_approx_normal((B, S + Tk), g) * 1.5, -5.0, 5.0)    # already normalised observations
    gt_action = _approx_normal((B, A), g) * 0.5
    noise = _approx_normal((B, E), g)
    progress = torch.zeros(NE, T, dtype=torch.int64)
    r = torch.randint(0, 1000, (NE, T + 1), generator=g)
    for e in range(NE):
        p = int(r[e, T]) % 40
        for t in range(T):
            if int(r[e, t]) < 60:                          # a reset inside the window
                p = 0
            progress[e, t] = p
            p += 1
    progress[0, :] = torch.arange(T)
    chk = sum(float(v.double().sum()) for v in sd.values()) + float(obs.double().sum()) + float(gt_action.double().sum()) + float(noise.double().sum())
    return sd, dict(obs=obs, gt_action=gt_action, noise=noise, progress=progress.reshape(B)), chk


# ----------------------------------------------------------------------------------------------------------------------
# Host-independent synthetic MotionLib tables + step inputs (BASELINE configs C2 / C4 sized parity fixtures): built from
# integer draws and single IEEE elementwise ops only (no reductions, no libm), so every host regenerates them bit for bit;
# fixtures store a float64 checksum.  Used by tests/golden/make_golden_step4096.py and the GPU tests.
# ----------------------------------------------------------------------------------------------------------------------
def _unit_quat(q):
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    n = torch.sqrt((x * x + y * y) + (z * z + w * w))
    return q / n.unsqueeze(-1)


def exact_tables(num_motions, seed=5, min_frames=5, max_frames=300, spread=230, fps=30.0):
    """oracle MotionTables with clip lengths from integer draws; unit quaternions (nearby frames), smooth-ish positions.
    fps: one rate, or a sequence of per-clip rates (clip_rates); the rates change only lengths, dt and fps."""
    from oracle.pulse_oracle import MotionTables
    g = torch.Generator().manual_seed(seed)
    nf = torch.randint(min_frames, min_frames + spread, (num_motions,), generator=g).clamp(max=max_frames)
    nf[:3] = torch.tensor([2, 5, max_frames])[: min(3, num_motions)]
    F = int(nf.sum())
    rep = lambda x: x.repeat_interleave(nf, dim=0)
    grs = _unit_quat(rep(_approx_normal((num_motions, 24, 4), g)) + 0.15 * _approx_normal((F, 24, 4), g))
    lrs = _unit_quat(rep(_approx_normal((num_motions, 24, 4), g)) + 0.15 * _approx_normal((F, 24, 4), g))
    gts = rep(_approx_normal((num_motions, 24, 3), g) * 0.4 + torch.tensor([0.0, 0.0, 0.9])) + 0.05 * _approx_normal((F, 24, 3), g)
    gvs, gavs, dvs = _approx_normal((F, 24, 3), g), _approx_normal((F, 24, 3), g), _approx_normal((F, 23, 3), g)
    aa = _approx_normal((F, 72), g)
    starts = torch.cumsum(nf, 0) - nf
    rates = clip_rates(fps, num_motions)
    lengths = ((nf - 1).double() * (1.0 / rates)).float()
    dt = (1.0 / rates).float()
    return MotionTables(gts=gts, grs=grs, lrs=lrs, gvs=gvs, gavs=gavs, dvs=dvs, motion_aa=aa, lengths=lengths, num_frames=nf, dt=dt,
                        length_starts=starts, fps=rates.float(), motion_bodies=torch.zeros(num_motions, 17),
                        motion_limb_weights=torch.zeros(num_motions, 10))


def exact_step_inputs(tb, n_envs, seed=6):
    """Simulator state NEAR the frames the step will query (so rewards are non-trivial and a fraction of the envs terminates),
    without calling any blend code: body j of env e = frame row (start frame + progress) of its clip + integer-exact noise."""
    g = torch.Generator().manual_seed(seed)
    M = tb.num_motions
    motion_ids = torch.arange(n_envs) % M
    nf = tb.num_frames[motion_ids]
    progress = torch.randint(0, 40, (n_envs,), generator=g)
    progress[:6] = torch.arange(6)[: min(6, n_envs)]
    f_start = torch.div(torch.randint(0, 1 << 20, (n_envs,), generator=g) * nf, 1 << 20, rounding_mode="floor")   # start frame in [0, nf)
    start = f_start.float() * (1.0 / 30)           # sample_time_interval's grid: k * fp32(1/30)... as the reference computes it
    start = (f_start.double() * (1.0 / 30)).float()
    start_off = torch.zeros(n_envs)
    goff = torch.zeros(n_envs, 3)
    goff[::4, :2] = _approx_normal(((n_envs + 3) // 4, 2), g)
    cycle = torch.zeros(n_envs, dtype=torch.int32)
    cycle[::7] = 5
    row = tb.length_starts[motion_ids] + torch.minimum(f_start + progress, nf - 1)
    amp = torch.full((n_envs, 1, 1), 0.03)
    amp[::5] = 0.12
    body_pos = tb.gts[row] + goff.unsqueeze(1) + amp * _approx_normal((n_envs, 24, 3), g)
    body_rot = _unit_quat(tb.grs[row] + 0.07 * _approx_normal((n_envs, 24, 4), g))
    body_vel = tb.gvs[row] + 0.5 * _approx_normal((n_envs, 24, 3), g)
    body_ang = tb.gavs[row] + 0.5 * _approx_normal((n_envs, 24, 3), g)
    z = {
        "motion_ids": motion_ids, "progress_buf": progress, "start_times": start, "start_offset": start_off, "global_offset": goff,
        "cycle_counter": cycle, "body_state": torch.cat([body_pos, body_rot, body_vel, body_ang], dim=-1).contiguous(),
        "dof_pos": 0.3 * _approx_normal((n_envs, 69), g), "dof_vel": _approx_normal((n_envs, 69), g),
        "dof_force": 30 * _approx_normal((n_envs, 69), g), "reset_buf_in": torch.zeros(n_envs, dtype=torch.long),
    }
    chk = float(tb.gts.double().sum() + tb.grs.double().sum() + tb.gvs.double().sum() + tb.lrs.double().sum()) \
        + sum(float(v.double().sum()) for v in z.values())
    return z, chk
