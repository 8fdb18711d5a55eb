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
import math

import numpy as np
import pytest
from twin import (ARM_MASK, BODY_BITS, BUILDS_OF, FOLDED, NOISE, SUB, UPPER_BITS, IterationBand, compare_control_steps,
                  compare_substeps, force_build, generic_path, limits, make_env, make_oracle, quat, rot, violated)

N = 37


def _kw(mark, terrain, sub=True, build=None):
    """The keywords of a scenario batch, the same for the GPU env and its oracle; the sensor build: observation noise only."""
    kw = dict(signal_type="ik", terrain_type=terrain, num_fields=4, mark=mark, seed=21, target_position=2.0, backwards=False)
    if sub:
        kw.update(SUB)
    if build == "sensor":
        kw["observation_noise_stdev"] = NOISE
    return kw


def _knees_ok(m, v):
    return any(v[3 * l:3 * l + 3].any() and (m >> (1 + 2 * l)) & 1 and (m >> (2 + 2 * l)) & 1 for l in range(4))


# what the start state of each scenario must exercise on the oracle: f(contact mask of its first sub-step, violated limits)
WANT = {"stand": lambda m, v: not (m & (BODY_BITS | ARM_MASK)) and v[:12].reshape(4, 3).sum(1).max() < 2,
        "back": lambda m, v: m & 1,                                 # base / chassis box (lane-0 rows 3-5)
        "side": lambda m, v: m & UPPER_BITS,                        # shoulder or leg box (rows 6-8)
        "tumble": lambda m, v: m & BODY_BITS,                       # contacts that come and go between sub-steps
        "nose": lambda m, v: m & BODY_BITS,
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
    o = make_oracle("walk", N, **_kw(mark, terrain))
    o.reset()
    s0 = [o.state(i) for i in range(N)]
    lo, hi = limits(mark)
    rng = np.random.default_rng(3)
    st, drop = [], {}
    for i, sid in enumerate(ids):
        c = ids[:i].count(sid)
        s = {k: np.array(v, dtype=np.float64) for k, v in s0[i].items()}
        if sid in DROPS or sid in ("deep", "knees"):
            r, p, dz, lin, ang = DROPS["back" if sid == "deep" else sid] if sid != "knees" else (0.02, 0.015, -0.165, (0, 0, -0.3), (0, 0, 0))
            s["pos"][2] += dz
            s["quat"] = quat(r + 0.004 * c, p + 0.003 * c, 0.02)
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
        o.set_state(i, st[i])
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


def _base_depth(states):
    """Depth of the deepest base / chassis box corner below z = 0 (flat ground)."""
    from rex_gym_b200.model_tables import load_model_json
    pts = np.concatenate([np.asarray(s["points"]).reshape(-1, 3) for s in load_model_json("base")["bodies"][0]["shapes"]])
    out = []
    for p, q in zip(states["pos"], states["quat"]):
        out.append((pts @ rot(q).T + p)[:, 2].min())
    return np.array(out)


@pytest.mark.parametrize("mark", ["base", "arm"])
@pytest.mark.parametrize("terrain", ["plane", "random"])
def test_scenarios_reach_the_generic_rows(mark, terrain):
    """CPU: the start state of every scenario, one sub-step on the oracle, contains the contact groups / limit rows it is there
    for (WANT), and every scenario but 'stand' takes the generic path."""
    ids, st = _batch(mark, terrain)
    o = make_oracle("walk", N, **_kw(mark, terrain))
    o.reset()
    for i in range(N):
        o.set_state(i, {k: v[i] for k, v in st.items()})
    viol = violated(st["q"], mark)
    o.step(np.zeros((N, o.A), np.float32))
    mask = np.array([o.env(i).contact_mask for i in range(N)])
    for i, sid in enumerate(ids):
        assert WANT[sid](mask[i], viol[i]), (i, sid, bin(mask[i]), viol[i].astype(int))
    np.testing.assert_array_equal(generic_path(mask, viol), [sid != "stand" for sid in ids])
    assert sum(o.env(i).limit_rows for i in range(N)) == viol.sum()
    if terrain == "plane":
        d = _base_depth(st)[[sid == "deep" for sid in ids]]
        assert (d < -0.04).all(), d                         # pen <= -0.04: no positional correction
    assert len(set(ids)) == (12 if mark == "arm" else 9)


CONFIGS = [(m, t, b) for m in ("base", "arm") for t in ("plane", "random") for b in BUILDS_OF[m]]


@pytest.mark.gpu
@pytest.mark.parametrize("mark,terrain,build", CONFIGS, ids=["-".join(c) for c in CONFIGS])
def test_generic_substeps_against_the_oracle(monkeypatch, mark, terrain, build):
    """One control step = one physics sub-step (control_time_step 1 ms, action_repeat 1, 60 PGS iterations), 30 of them, the
    CUDA state re-synchronised to the oracle before each.  Per sub-step: the solver cost decodes exactly (// 64: the generic
    path ran, % 64: PGS iterations) -- the path is the oracle's predicate on its contact mask and the violated limits, the
    iteration count lies in the range the oracle spans over early-out thresholds 0.8-1.2e-7 in its fp64 and fp32 builds; the
    contact mask equals the oracle's on every group; q and pos meet test_one_step_is_tight's bounds (90th percentile 2e-5 rad /
    2e-6 m, none beyond 3e-3).
    Measured on an H100 SXM (all 1110 samples of a configuration; the three builds of a terrain agree bit for bit):
      flat ground      q median 9e-8, p90 2-4e-7, max 2.6e-6 rad; pos median 3e-9, p90 1e-8, max 3e-8 m; iterations all in the band
      heightfield      q median 9e-8, p90 2e-7, max 4.4e-6 rad;   pos max 3e-8 m;                        all in the band
      arm, heightfield q median 1.5e-7, p90 1.1e-6, max 6.4e-4 rad; pos max 1.8e-6 m; one sample one iteration off the band
    so the iteration band allows 3 samples out of it."""
    force_build(monkeypatch, build)
    kw = _kw(mark, terrain, build=build)
    env, ora = make_env("walk", N, **kw), make_oracle("walk", N, **kw)
    band = IterationBand(lambda **b: make_oracle("walk", N, **kw, **b))
    env.reset(); ora.reset(); band.reset()
    ids, st = _batch(mark, terrain)
    eq, ep, off_band, generic_steps, _, _ = compare_substeps(env, ora, band, st, build, ids)
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
    force_build(monkeypatch, build)
    kw = _kw(mark, terrain, sub=False, build=build)
    env, ora = make_env("walk", N, **kw), make_oracle("walk", N, **kw)
    env.reset(); ora.reset()
    ids, st = _batch(mark, terrain)
    eqs, eps_, _ = compare_control_steps(env, ora, st, build, ids, q90=1e-3, p90=1e-3, qmax=5e-2, pmax=5e-3)
    print("generic control steps q (median, p90, max), pos (median, p90, max):",
          (np.median(eqs), np.percentile(eqs, 90), eqs.max(), np.median(eps_), np.percentile(eps_, 90), eps_.max()))
    assert env.check_errors() == 0
    env.close()
