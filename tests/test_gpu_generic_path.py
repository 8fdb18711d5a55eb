"""The generic solver path of physics_substep against the fp64 oracle, in every build of the step kernel.

physics_substep (rex_gym_b200/csrc/rexsim_kernel.cu) solves the foot contacts, one joint limit per leg and up to ARM_KA arm limits
in its fast path; everything else takes the generic path: body-box contacts (base and chassis on lane 0, shoulder and leg boxes on
every lane), arm-link contacts, two or three violated limits in one leg, more than ARM_KA violated arm limits.  Walking, galloping
and turning never get there (a falling robot terminates at 32 degrees before a box touches), so the states here are built on
purpose: each scenario is a pose the CPU oracle drops until the wanted contacts exist, and the oracle's state at that moment is
the start state of both sides (set_state on the GPU, the RexoEnv struct on the oracle).

test_scenarios_reach_the_generic_rows (CPU) pins what every scenario exercises, so the GPU tests cannot go vacuous when the model
or a constant moves.  The GPU tests run each scenario (with jittered copies and standing envs, 37 envs: envs on the generic path,
on the fast path and without contact share warps) in {small, big, sensor} x {plane, random} and, with the arm, {small, sensor} x
{plane, random}.
"""
import ctypes
import math

import numpy as np
import pytest

from test_gpu_builds import BUILDS, _launched

TOES = (2, 4, 6, 8)
UPPER = (1, 3, 5, 7)
ARM_BITS = tuple(range(9, 15))
HOLD = (0.8e-7, 0.9e-7, 1e-7, 1.1e-7, 1.2e-7)           # test_gpu_parity.HOLD_THRESHOLDS
SUB = dict(control_time_step=0.001, action_repeat=1, solver_iterations=60)   # one control step = one physics sub-step
NOISE = (0.01, 0.05, 0.1, 0.02, 0.1)                     # the sensor build, with zero latencies
N = 37


def _quat(r, p, y):
    cr, sr, cp, sp, cy, sy = (f(0.5 * a) for a in (r, p, y) for f in (math.cos, math.sin))
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


def _oracle(mark, terrain, n, sub=True, **kw):
    from oracle.oracle import OracleSim
    if sub:
        kw.update(SUB)
    return OracleSim(n, "walk", "ik", terrain=terrain, nfields=4 if terrain == "random" else 0, mark=mark, seed=21,
                     target_position=2.0, backwards=False, **kw)


def _write(ora, i, st):
    """Write a physical state into the oracle's env struct (the oracle has no set_state)."""
    e = ora.env(i)
    for k, m in (("pos", 3), ("quat", 4), ("linvel", 3), ("angvel", 3)):
        for a in range(m):
            getattr(e, k)[a] = float(st[k][a])
    for j in range(len(st["q"])):
        e.q[j], e.qd[j] = float(st["q"][j]), float(st["qd"][j])


def _limits(mark):
    from oracle.oracle import load_model
    m, _ = load_model(mark)
    return np.array([m.lower[j + 1] for j in range(m.ndof)]), np.array([m.upper[j + 1] for j in range(m.ndof)])


def _violated(q, mark):
    """Violated joint limits per env as the fp32 kernel sees them: [N][ndof] bool."""
    lo, hi = _limits(mark)
    q = np.asarray(q, np.float32)
    return (q - lo.astype(np.float32) <= 0) | (hi.astype(np.float32) - q <= 0)


def _generic(mask, viol):
    """The generic-path predicate: a body or arm contact, two or more limits in one leg, more than three arm limits."""
    body = (mask & ((1 << 0) | sum(1 << b for b in UPPER) | sum(1 << b for b in ARM_BITS))) != 0
    legs = viol[:, :12].reshape(-1, 4, 3).sum(2).max(1) >= 2
    arm = viol[:, 12:].sum(1) > 3 if viol.shape[1] > 12 else np.zeros(len(viol), bool)
    return body | legs | arm


BODY = (1 << 0) | sum(1 << b for b in UPPER)
ARM_MASK = sum(1 << b for b in ARM_BITS)


def _knees_ok(m, v):
    return any(v[3 * l:3 * l + 3].any() and (m >> (1 + 2 * l)) & 1 and (m >> (2 + 2 * l)) & 1 for l in range(4))


# what the start state of each scenario must exercise on the oracle: f(contact mask of its first sub-step, violated limits)
WANT = {"stand": lambda m, v: not (m & (BODY | ARM_MASK)) and v[:12].reshape(4, 3).sum(1).max() < 2,
        "back": lambda m, v: m & 1,                                 # base / chassis box (lane-0 rows 3-5)
        "side": lambda m, v: m & (BODY ^ 1),                        # shoulder or leg box (rows 6-8)
        "tumble": lambda m, v: m & BODY,                            # contacts that come and go between sub-steps
        "nose": lambda m, v: m & BODY,
        "knees": _knees_ok,                                         # limit, upper and foot rows in one lane: all 12 rows
        "deep": lambda m, v: m & 1,                                 # + a base corner 5 cm deep: the split-impulse branch
        "two-air": lambda m, v: v[:12].reshape(4, 3).sum(1).max() >= 2,
        "two-stand": lambda m, v: v[:12].reshape(4, 3).sum(1).max() >= 2,
        "arm-back": lambda m, v: m & ARM_MASK,                      # arm-link contacts
        "arm-side": lambda m, v: m & ARM_MASK,
        "arm-limits": lambda m, v: v[12:].sum() > 3}                # more than ARM_KA arm limit rows
# dropped scenarios: roll, pitch, height above the settled base, linear and angular velocity
DROPS = {"back": (math.pi + 0.04, 0.03, 0.1, (0, 0, 0), (0, 0, 0)), "side": (math.pi / 2 + 0.05, 0.02, 0.1, (0, 0, 0), (0, 0, 0)),
         "tumble": (0.9, 0.4, 0.15, (0.5, 0, 0), (3.0, 0, 0)), "nose": (0.03, 1.2, 0.1, (0, 0, 0), (0, 0, 0)),
         "arm-back": (math.pi + 0.04, 0.03, 0.1, (0, 0, 0), (0, 0, 0)), "arm-side": (math.pi / 2 + 0.05, 0.02, 0.1, (0, 0, 0), (0, 0, 0))}
FOLDED = np.array([-0.42, -1.51, 2.70, 0.42, -1.51, 2.70, -0.44, -1.49, 2.69, 0.44, -1.49, 2.69])   # standup's settled legs


def _layout(mark):
    sc = [k for k in WANT if k != "stand" and (mark == "arm" or not k.startswith("arm"))]
    return ["stand"] * 3 + [sc[i % len(sc)] for i in range(N - 3)]


def _batch(mark, terrain):
    """-> (scenario id per env, start state {key: [N][...]}).  Every env is built in its own slot of an N-env oracle (the
    heightfield of an env depends on its index); copy c of a scenario is tilted c x 4 mrad further than copy 0."""
    key = (mark, terrain)
    if key in _CACHE:
        return _CACHE[key]
    ids = _layout(mark)
    o = _oracle(mark, terrain, N)
    o.reset()
    s0 = [o.state(i) for i in range(N)]
    lo, hi = _limits(mark)
    rng = np.random.default_rng(3)
    st, drop = [], {}
    for i, sid in enumerate(ids):
        c = ids[:i].count(sid)
        s = {k: np.array(v, dtype=np.float64) for k, v in s0[i].items()}
        if sid in DROPS or sid in ("deep", "knees"):
            r, p, dz, lin, ang = DROPS["back" if sid == "deep" else sid] if sid != "knees" else (0.02, 0.015, -0.165, (0, 0, -0.3), (0, 0, 0))
            s["pos"][2] += dz
            s["quat"] = _quat(r + 0.004 * c, p + 0.003 * c, 0.02)
            s["linvel"], s["angvel"], s["qd"] = np.array(lin, float), np.array(ang, float), np.zeros_like(s["qd"])
            if sid == "knees":
                s["q"][:12] = FOLDED + np.repeat([0.0, 4e-3, 8e-3, 12e-3], 3) + 1e-3 * c
            else:
                drop[i] = sid
        elif sid in ("two-air", "two-stand"):
            if sid == "two-air":
                s["pos"][2] = 0.4
            for l in rng.choice(4, size=1 + c % 3, replace=False):
                s["q"][3 * l + 1] = hi[3 * l + 1] + rng.uniform(0.002, 0.03)     # leg joint past its upper limit
                s["q"][3 * l + 2] = lo[3 * l + 2] - rng.uniform(0.002, 0.03)     # foot joint past its lower limit
                if (c + l) % 2:
                    s["q"][3 * l] = (hi[3 * l] + rng.uniform(0.002, 0.03)) * (1 if l % 2 else -1)
                s["qd"][3 * l:3 * l + 3] = rng.uniform(-1.0, 1.0, 3)
        elif sid == "arm-limits":                          # the rest pose already holds joints 0, 1, 4 past their limits
            s["q"][14] = hi[14] + 0.01 + 0.002 * c
            s["q"][15] = lo[15] - 0.02
            if c % 2 == 0:
                s["q"][17] = hi[17] + 0.015
        st.append(s)
    # drop every dropped env until its scenario's contacts exist; its start state is the state before that sub-step
    for i in drop:
        _write(o, i, st[i])
    pending = set(drop)
    for _ in range(600):
        if not pending:
            break
        prev = {i: o.state(i) for i in pending}
        o.step(np.zeros((N, o.A), np.float32))
        for i in list(pending):
            m = o.env(i).contact_mask
            if WANT[drop[i]](m, np.zeros(18, bool)):
                st[i] = prev[i]
                pending.discard(i)
    assert not pending, [ids[i] for i in pending]
    for i, sid in enumerate(ids):
        if sid == "deep":
            st[i]["pos"][2] -= 0.05
    out = ids, {k: np.stack([s[k] for s in st]) for k in st[0]}
    _CACHE[key] = out
    return out


_CACHE = {}


def _start(ora, states):
    for i in range(ora.N):
        _write(ora, i, {k: v[i] for k, v in states.items()})


def _base_depth(states):
    """Depth of the deepest base / chassis box corner below z = 0 (flat ground)."""
    from rex_gym_b200.model_tables import load_model_json
    pts = np.concatenate([np.asarray(s["points"]).reshape(-1, 3) for s in load_model_json("base")["bodies"][0]["shapes"]])
    out = []
    for p, q in zip(states["pos"], states["quat"]):
        x, y, z, w = q
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
        out.append((pts @ R.T + p)[:, 2].min())
    return np.array(out)


@pytest.mark.parametrize("mark", ["base", "arm"])
@pytest.mark.parametrize("terrain", ["plane", "random"])
def test_scenarios_reach_the_generic_rows(mark, terrain):
    """CPU: the start state of every scenario, one sub-step on the oracle, contains the contact groups / limit rows it is there
    for (WANT), and every scenario but 'stand' takes the generic path."""
    ids, st = _batch(mark, terrain)
    o = _oracle(mark, terrain, N)
    o.reset()
    _start(o, st)
    viol = _violated(st["q"], mark)
    o.step(np.zeros((N, o.A), np.float32))
    mask = np.array([o.env(i).contact_mask for i in range(N)])
    for i, sid in enumerate(ids):
        assert WANT[sid](mask[i], viol[i]), (i, sid, bin(mask[i]), viol[i].astype(int))
    np.testing.assert_array_equal(_generic(mask, viol), [sid != "stand" for sid in ids])
    assert sum(o.env(i).limit_rows for i in range(N)) == viol.sum()
    if terrain == "plane":
        d = _base_depth(st)[[sid == "deep" for sid in ids]]
        assert (d < -0.04).all(), d                         # pen <= -0.04: no positional correction
    assert len(set(ids)) == (12 if mark == "arm" else 9)


CONFIGS = [(m, t, b) for m, builds in (("base", ("small", "big", "sensor")), ("arm", ("small", "sensor")))
           for t in ("plane", "random") for b in builds]


def _gpu_env(mark, terrain, build, monkeypatch, sub=True):
    import rex_gym_b200 as R
    if build == "sensor":
        monkeypatch.delenv("REXSIM_FORCE_BUILD", raising=False)
    else:
        monkeypatch.setenv("REXSIM_FORCE_BUILD", build)
    kw = dict(SUB) if sub else {}
    if build == "sensor":
        kw["observation_noise_stdev"] = NOISE
    env = R.BatchedRexEnv(task="walk", num_envs=N, signal_type="ik", terrain_type=terrain, num_fields=4, mark=mark, seed=21,
                          target_position=2.0, backwards=False, **kw)
    okw = {"observation_noise_stdev": NOISE} if build == "sensor" else {}
    return env, okw


def _cost(env):
    import torch
    from rex_gym_b200.envs.batched_env import _DevArray
    p = ctypes.c_void_p()
    assert env._L.rexsim_solver_cost(env._h, ctypes.byref(p)) == 0
    return torch.as_tensor(_DevArray(p.value, (env.num_envs,), "<i4", env), device="cuda").cpu().numpy().copy()


def _set(env, s):
    env.set_state(s["pos"], s["quat"], s["linvel"], s["angvel"], s["q"], s["qd"])


def _ostate(ora):
    from test_gpu_parity import _oracle_state
    return _oracle_state(ora, ora.N)


@pytest.mark.gpu
@pytest.mark.parametrize("mark,terrain,build", CONFIGS, ids=["-".join(c) for c in CONFIGS])
def test_generic_substeps_against_the_oracle(monkeypatch, mark, terrain, build):
    """One control step = one physics sub-step (control_time_step 1 ms, action_repeat 1, 60 PGS iterations), 30 of them, the
    CUDA state re-synchronised to the oracle before each.  Per sub-step: rexsim_solver_cost decodes exactly (// 64: the generic
    path ran, % 64: PGS iterations) -- the path is the oracle's predicate on its contact mask and the violated limits, the
    iteration count lies in the range the oracle spans over early-out thresholds 0.8-1.2e-7 in its fp64 and fp32 builds; the
    contact mask equals the oracle's on every group; q and pos meet test_one_step_is_tight's bounds (90th percentile 2e-5 rad /
    2e-6 m, none beyond 3e-3).
    Measured on an H100 SXM (all 1110 samples of a configuration; the three builds of a terrain agree bit for bit):
      flat ground      q median 9e-8, p90 2-4e-7, max 2.6e-6 rad; pos median 3e-9, p90 1e-8, max 3e-8 m; iterations all in the band
      heightfield      q median 9e-8, p90 2e-7, max 4.4e-6 rad;   pos max 3e-8 m;                        all in the band
      arm, heightfield q median 1.5e-7, p90 1.1e-6, max 6.4e-4 rad; pos max 1.8e-6 m; one sample one iteration off the band
    so the iteration band allows 3 samples out of it."""
    env, okw = _gpu_env(mark, terrain, build, monkeypatch)
    ora = _oracle(mark, terrain, N, **okw)
    band = [_oracle(mark, terrain, N, residual_threshold=t, f32=f, **okw) for t in HOLD for f in (False, True)]
    env.reset(); ora.reset()
    for b in band:
        b.reset()
    ids, st = _batch(mark, terrain)
    _start(ora, st)
    full = 0x7FFF if mark == "arm" else 0x1FF
    rng = np.random.default_rng(7)
    eq, ep, off_band, generic_steps = [], [], 0, 0
    for k in range(30):
        so = _ostate(ora)
        _set(env, so)
        for b in band:
            _start(b, so)
        viol = _violated(so["q"], mark)
        a = rng.uniform(-0.4, 0.4, size=(N, env.action_dim)).astype(np.float32)
        env.step(a)
        assert _launched(env) == BUILDS[build], _launched(env)
        ora.step(a)
        its = []
        for b in band:
            b.step(a)
            its.append([b.env(i).solver_iters for i in range(N)])
        cost, sg = _cost(env), env.get_state()
        mask = np.array([ora.env(i).contact_mask for i in range(N)]) & full
        np.testing.assert_array_equal(sg["contact_mask"] & full, mask, err_msg=f"contact mask, sub-step {k}")
        gen = _generic(mask, viol)
        np.testing.assert_array_equal(cost >= 64, gen, err_msg=f"solver path, sub-step {k}")
        generic_steps += gen.sum()
        lo_it, hi_it = np.min(its, 0), np.max(its, 0)
        off_band += ((cost % 64 < lo_it) | (cost % 64 > hi_it)).sum()
        s2 = _ostate(ora)
        eq.append(np.abs(sg["q"] - s2["q"]).max(1)); ep.append(np.abs(sg["pos"] - s2["pos"]).max(1))
    eq, ep = np.concatenate(eq), np.concatenate(ep)
    stats = (np.median(eq), np.percentile(eq, 90), eq.max(), np.median(ep), np.percentile(ep, 90), ep.max(), off_band)
    print("generic sub-steps q (median, p90, max), pos (median, p90, max), iterations off the band:", stats)
    assert generic_steps >= 30 * (N - 3) * 0.5, generic_steps
    assert off_band <= 3, stats
    assert np.percentile(eq, 90) < 2e-5 and np.percentile(ep, 90) < 2e-6 and eq.max() < 3e-3 and ep.max() < 3e-3, stats
    assert env.check_errors() == 0
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mark,terrain,build", CONFIGS, ids=["-".join(c) for c in CONFIGS])
def test_generic_control_steps_against_the_oracle(monkeypatch, mark, terrain, build):
    """The task configuration (5 sub-steps per control step): 20 control steps of random actions inside walk-ik's bound from the
    scenario states, re-synchronised every 5, within test_free_running_rollout's strict window (90th percentile of the envs
    1e-3 rad / 1e-3 m, none beyond 5e-2 / 5e-3); every output finite, no error bit (no TILE_MISS, no non-finite).
    Measured on an H100 SXM over the 740 samples of a configuration (q median / p90 / max in rad, pos max in m):
      flat ground 2.5e-7 / 7e-7 / 3.1e-5, 3.7e-7;  heightfield 3.1e-7 / 2.1e-6 / 6.1e-4, 4.1e-6;
      arm, flat   3.8e-7 / 2.2e-6 / 7.0e-4, 4.2e-6;  arm, heightfield 7.0e-7 / 7.4e-6 / 3.1e-3, 1.0e-4."""
    env, okw = _gpu_env(mark, terrain, build, monkeypatch, sub=False)
    ora = _oracle(mark, terrain, N, sub=False, **okw)
    env.reset(); ora.reset()
    ids, st = _batch(mark, terrain)
    _start(ora, st)
    rng = np.random.default_rng(9)
    eqs, eps_ = [], []
    for k in range(20):
        if k % 5 == 0:
            _set(env, _ostate(ora))
        a = rng.uniform(-0.4, 0.4, size=(N, env.action_dim)).astype(np.float32)
        og, rg, _, _ = env.step(a)
        assert _launched(env) == BUILDS[build], _launched(env)
        ora.step(a)
        assert np.isfinite(og).all() and np.isfinite(rg).all()
        sg, so = env.get_state(), _ostate(ora)
        assert all(np.isfinite(v).all() for v in sg.values())
        eq = np.abs(sg["q"] - so["q"]).max(1)
        ep = np.abs(sg["pos"] - so["pos"]).max(1)
        eqs.append(eq); eps_.append(ep)
        assert np.percentile(eq, 90) < 1e-3 and np.percentile(ep, 90) < 1e-3, f"step {k}: {np.percentile(eq, 90):.2e} {np.percentile(ep, 90):.2e}"
        assert eq.max() < 5e-2 and ep.max() < 5e-3, f"step {k}: {eq.max():.2e} {ep.max():.2e} in {ids[int(np.argmax(eq))]}"
    eqs, eps_ = np.concatenate(eqs), np.concatenate(eps_)
    print("generic control steps q (median, p90, max), pos (median, p90, max):",
          (np.median(eqs), np.percentile(eqs, 90), eqs.max(), np.median(eps_), np.percentile(eps_, 90), eps_.max()))
    assert env.check_errors() == 0
    env.close()
