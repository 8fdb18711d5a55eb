"""Final observations and gym's TimeLimit key from auto-resetting steps, and the bootstrap of truncated episodes.

An auto-resetting step (BatchedRexEnv(auto_reset=True), every Rollout) replaces a done env's observation with the first one of
its next episode.  final_observation=True keeps what the reference's BatchEnv.step returns before the reset at the top of the
next iteration (in_graph_batch_env.py:71-113, simulate.py:67-75), and the time-limit byte behind gym 0.17.1's
info['TimeLimit.truncated'].  The checks: every step-kernel instance against an auto_reset=False twin that resets its done envs
by hand, the limit byte against its definition and the task's restated termination, the host path against the device path on
both sides of the zero-copy limit, graph rollouts against the loop and a replay, and the bootstrap scan against an fp64
restatement.
"""
import types

import numpy as np
import pytest

from oracle import agent_oracle as AO

# ---- gym 0.17.1 wrappers/time_limit.py, restated (gym is not a dependency) ------------------------------------------------
#     def step(self, action):
#         observation, reward, done, info = self.env.step(action)
#         self._elapsed_steps += 1
#         if self._elapsed_steps >= self._max_episode_steps:
#             info['TimeLimit.truncated'] = not done
#             done = True
#         return observation, reward, done, info
def gym_time_limit(elapsed_steps, max_episode_steps, inner_done):
    """-> (done, info additions) of TimeLimit.step after the inner env returned `inner_done` at its step `elapsed_steps`."""
    info = {}
    if elapsed_steps >= max_episode_steps:
        info["TimeLimit.truncated"] = not inner_done
        inner_done = True
    return inner_done, info


def limit_byte(at_limit, ended):
    """The step kernel's time-limit byte: bit 0 the limit was reached, bit 1 the episode also ended otherwise."""
    return (1 if at_limit else 0) | (2 if ended else 0)


def gae_bootstrap_fp64(reward, value, done, truncated, final_value, discount, lam):
    """rexsim_gae_segments_bootstrap in fp64: agent_oracle.gae_segments, except that a done and truncated step bootstraps from
    final_value and cuts both chains there."""
    reward, value, final_value = (np.asarray(x, np.float64) for x in (reward, value, final_value))
    T, n = reward.shape
    nd = 1.0 - np.asarray(done, np.float64)
    cut = np.asarray(done, bool) & np.asarray(truncated, bool)
    ret, adv = np.zeros((T, n)), np.zeros((T, n))
    r_next, a_next, v_next = value[T].copy(), np.zeros(n), value[T].copy()
    for t in range(T - 1, -1, -1):
        delta = reward[t] + discount * v_next * nd[t] - value[t]
        a_next = np.where(cut[t], reward[t] + discount * final_value[t] - value[t], delta + discount * lam * nd[t] * a_next)
        r_next = np.where(cut[t], reward[t] + discount * final_value[t], reward[t] + discount * nd[t] * r_next)
        adv[t], ret[t] = a_next, r_next
        v_next = value[t]
    return ret, adv


# ---- CPU ------------------------------------------------------------------------------------------------------------------
def test_entry_points_are_declared_and_bound():
    import os
    import re
    from rex_gym_b200 import _capi
    inc = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include")
    src = open(os.path.join(inc, "rexsim.h")).read() + open(os.path.join(inc, "rexsim_agent.h")).read()
    for name, nargs in (("rexsim_step_final", 8), ("rexsim_host_final_bytes", 1), ("rexsim_step_host_final", 5),
                        ("rexsim_gae_segments_bootstrap", 12)):
        m = re.search(r"\b%s\s*\(([^)]*)\)" % name, src)
        assert m, name
        assert len(m.group(1).split(",")) == nargs == len(_capi.SIGNATURES[name][1]), name


@pytest.mark.parametrize("max_steps", [1, 7, 400])
def test_limit_byte_carries_gyms_key(max_steps):
    """The byte -> info mapping of _Info against the restated TimeLimit, for every step count around the limit and both inner
    outcomes (no device: a stand-in env hands _Info its commands and bytes)."""
    import torch
    from rex_gym_b200.envs.batched_env import _Info
    cases = [(k, ended) for k in range(1, max_steps + 3) for ended in (False, True)]
    n = len(cases)
    lim = np.array([limit_byte(k >= max_steps, ended) for k, ended in cases], np.uint8)
    env = types.SimpleNamespace(_nsteps=3, _final=object(), __len__=lambda: n,
                                last_command=lambda: torch.zeros((12, n)), limit_bytes=lambda: lim)
    info = _Info(env)
    for i, (k, ended) in enumerate(cases):
        done, extra = gym_time_limit(k, max_steps, ended)
        got = info[i]
        assert set(got) == {"action"} | set(extra), (k, ended, got)
        assert got.get("TimeLimit.truncated") == extra.get("TimeLimit.truncated")
        assert done == (ended or bool(lim[i] & 1))
    off = _Info(types.SimpleNamespace(_nsteps=3, _final=None, last_command=lambda: torch.zeros((12, n))))
    assert set(off[0]) == {"action"}


def test_bootstrap_restatement_is_the_plain_scan_without_truncations():
    rng = np.random.default_rng(0)
    T, n = 9, 6
    r, v, d = rng.normal(size=(T, n)), rng.normal(size=(T + 1, n)), rng.random((T, n)) < 0.3
    for got, want in zip(gae_bootstrap_fp64(r, v, d, np.zeros((T, n), bool), rng.normal(size=(T, n)), 0.9, 0.8),
                         AO.gae_segments(r, v, d, 0.9, 0.8)):
        np.testing.assert_array_equal(got, want)


# ---- GPU helpers ----------------------------------------------------------------------------------------------------------
def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _words(env):
    out = dict(state_f=_np(env._state_f), state_i=_np(env._state_i), cmd=_np(env.last_command()))
    if env._ring is not None:
        out["sensor_history"] = _np(env._ring)
    if env._episode is not None:
        out["episode_statistics"] = _np(env._episode["block"])
    for k, v in env._frames.items():
        out[k] = _np(v)
    return out


def _restate_cfg(env):
    """task_outputs.restate's configuration from the batch's own RexSimConfig, without the time limit: the task's termination."""
    c = env._cfg
    return types.SimpleNamespace(task=env.task, sig=env.signal_type, nm=env.num_motors, dt=c.sim_dt_d, backwards=c.backwards,
                                 w=(c.w_distance, c.w_energy, c.w_drift, c.w_shake), normalize=bool(c.normalize), max_steps=0,
                                 seed=c.seed, env_offset=c.env_offset, latency=c.control_latency, sd=np.array(c.noise_stdev[:5]),
                                 sensor=env._ring is not None)


SENTINEL = np.float32(-12345.5)


def _tip(env, envs, roll=1.0):
    """Roll the bases of `envs` by `roll` rad (walk: is_fallen once the up component drops below 0.85)."""
    from twin import quat, qmul
    st = env.get_state()
    for e in envs:
        st["quat"][e] = qmul(quat(roll, 0.0, 0.0), st["quat"][e])
    env.set_state(*(st[k] for k in ("pos", "quat", "linvel", "angvel", "q", "qd")))


from twin import BUILDS, INSTANCES, bound, force_build, instance_config, launched, row_id  # noqa: E402


# ---- GPU: every step-kernel instance against its explicitly resetting twin -----------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("row", INSTANCES, ids=[row_id(r) for r in INSTANCES])
def test_every_instance_keeps_the_twins_step_observation(row, monkeypatch):
    """Batch A auto-resets with final outputs on (device path); its twin B, same keywords with auto_reset=False (numpy path),
    resets exactly its done envs through reset(idx) after every step.  Bit for bit, every step: rewards, dones, every state
    word (SoA, sensor ring, episode books, frame buffers); A's final rows of done envs = B's step observation = B's own final
    rows; A's other final rows keep a sentinel; A's observation = B's after its resets; both limit bytes equal, bit 0 is
    env_step == max_episode_steps, bit 1 the task's termination restated from B's state words away from its margins."""
    import torch
    from task_outputs import kernel_ring, kernel_words, restate
    from twin import make_env
    task, sig, arm, terrain, build = row
    force_build(monkeypatch, build)
    i = INSTANCES.index(row)
    n, steps, max_steps = 37, 300, (7, 13)[i % 2]
    kw = dict(instance_config(row), max_episode_steps=max_steps, episode_statistics=True, normalize=(i // 2) % 2 == 0,
              final_observation=True)
    if i % 3 == 0:
        kw.update(frame_history=[0, 1, 2, 3], frame_delta=True)
    A, B = make_env(task, n, auto_reset=True, **kw), make_env(task, n, auto_reset=False, **kw)
    np.testing.assert_array_equal(_np(A.reset()), _np(B.reset()))
    cfg = _restate_cfg(B)
    rng = np.random.default_rng(100 + i)
    b = bound(task, sig) * (1.5 if kw["normalize"] else 1.0)
    ended = limited = checked = 0
    for k in range(steps):
        if k % 5 == 3:              # a few bases rolled over, in both twins: task endings before and on the limit step
            tip = rng.choice(n, size=4, replace=False)
            _tip(A, tip); _tip(B, tip)
        a = rng.uniform(-b, b, size=(n, A.action_dim)).astype(np.float32)
        A._final.fill_(float(SENTINEL)); A._limit.fill_(0xEE)
        oA, rA, dA, _ = A.step(torch.from_numpy(a).cuda())
        oB, rB, dB, _ = B.step(a)
        assert launched(A) == launched(B) == BUILDS[build]
        oA, rA, dA = _np(oA), _np(rA), _np(dA)
        np.testing.assert_array_equal(rA, rB, err_msg=f"reward, step {k}")
        np.testing.assert_array_equal(dA, dB, err_msg=f"done, step {k}")
        fA, lA = _np(A.final_observation()), _np(A.limit_bytes())
        np.testing.assert_array_equal(fA[dA], oB[dA], err_msg=f"final rows, step {k}")
        assert (fA[~dA] == SENTINEL).all(), f"untouched rows, step {k}"
        np.testing.assert_array_equal(B.final_observation()[dB], oB[dB], err_msg=f"auto_reset=False final rows, step {k}")
        np.testing.assert_array_equal(lA, B.limit_bytes(), err_msg=f"limit, step {k}")
        w = kernel_words(B)
        np.testing.assert_array_equal(lA & 1, w["env_step"] == max_steps, err_msg=f"bit 0, step {k}")
        assert ((lA & 1) != 0)[~dA].sum() == 0 and (lA <= 3).all()
        term = restate(cfg, w, kernel_ring(B))
        clear = term.done_margin > 1e-4
        np.testing.assert_array_equal(((lA & 2) != 0)[clear], term.done[clear], err_msg=f"bit 1, step {k}")
        checked += clear.sum()
        np.testing.assert_array_equal(((lA & 3) != 0), dA, err_msg=f"done = bit 0 | bit 1, step {k}")
        ended += dA.sum(); limited += (lA & 1).sum()
        idx = np.nonzero(dB)[0]
        if idx.size:
            oB = oB.copy()
            oB[idx] = B.reset(idx)
        np.testing.assert_array_equal(oA, oB, err_msg=f"obs after the resets, step {k}")
        wA, wB = _words(A), _words(B)
        for key in wA:
            np.testing.assert_array_equal(wA[key], wB[key], err_msg=f"{key}, step {k}")
    assert limited > n and checked > 0.9 * n * steps
    if task != "poses":
        assert ended > limited                                 # some episodes ended by the task
    A.close(); B.close()


# ---- GPU: the limit byte and gym's key where a task ending falls on the limit step ---------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("path", ["device", "numpy", "single"])
def test_info_carries_gyms_key_exactly_on_the_limit_steps(path):
    """walk-ik, max_episode_steps=5: envs tipped before step 5 fall on the limit step (key False), envs tipped before step 3
    fall before it (no key), the rest are cut by the limit (key True); poses never terminates (key True at every limit).
    info[i] is gym 0.17.1's, on the device and numpy paths and through SingleRexEnv; with the switch off it is
    {'action': ...}."""
    import torch
    from rex_gym_b200.envs.single_env import RexPosesEnv, RexWalkEnv
    from twin import make_env
    kw = dict(signal_type="ik", seed=3, max_episode_steps=5, auto_reset=True, target_position=2.0, backwards=False)
    for task, single in (("walk", RexWalkEnv), ("poses", RexPosesEnv)):
        n = 1 if path == "single" else 12
        env = single(final_observation=True, **kw) if path == "single" else make_env(task, n, final_observation=True, **kw)
        batch = env._batch if path == "single" else env
        off = make_env(task, n, **kw)
        env.reset(); off.reset()
        elapsed, episode = np.zeros(n, int), np.zeros(n, int)
        seen = set()
        for k in range(15):
            if task == "walk":
                # episode e of env i: (i + e) % 3 == 0 tipped before its step 3, == 1 before its step 5 (the limit step)
                sel = (np.arange(n) + episode) % 3
                tip = np.nonzero(((sel == 0) & (elapsed == 2)) | ((sel == 1) & (elapsed == 4)))[0]
                if tip.size:
                    _tip(batch, tip); _tip(off, tip)
            a = np.zeros((n, batch.action_dim), np.float32)
            if path == "single":
                _, _, d, info = env.step(a[0])
                d, infos = np.array([d]), [info]
            elif path == "device":
                _, _, d, info = env.step(torch.from_numpy(a).cuda())
                d, infos = _np(d), [info[i] for i in range(n)]
            else:
                _, _, d, info = env.step(a)
                infos = [info[i] for i in range(n)]
            _, _, d_off, info_off = off.step(a)
            np.testing.assert_array_equal(d, d_off)
            assert all(info_off[i].keys() == {"action"} for i in range(n))
            elapsed += 1
            lim = _np(batch.limit_bytes())
            for i in range(n):
                inner = bool(lim[i] & 2)
                done, extra = gym_time_limit(elapsed[i], 5, inner)
                assert done == bool(d[i]) and set(infos[i]) == {"action"} | set(extra), (task, k, i, infos[i], lim[i])
                assert infos[i].get("TimeLimit.truncated") == extra.get("TimeLimit.truncated")
                np.testing.assert_array_equal(infos[i]["action"], info_off[i]["action"])
                if extra:
                    seen.add(extra["TimeLimit.truncated"])
                elif done:
                    seen.add("terminated")
            np.testing.assert_array_equal(_np(batch.truncated()), lim == 1)
            elapsed[d] = 0
            episode[d] += 1
        assert seen == ({True, False, "terminated"} if task == "walk" else {True}), (task, seen)
        env.close(); off.close()


# ---- GPU: host path against device path ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [16384, 16385], ids=["zero-copy", "staged"])
def test_host_path_returns_the_device_bytes(n):
    """The numpy path (rexsim_step_host_final) against the device path, bit for bit, on both sides of the zero-copy limit:
    observations, rewards, dones, final rows (whole buffers, ended or not) and limit bytes.  With auto_reset=False the final
    rows of done envs are their observation rows.  An out-of-range device reset index still only raises IndexError."""
    import torch
    from twin import make_env
    kw = dict(seed=4, normalize=True, max_episode_steps=7, frame_history=[0, 2, 1, 2], frame_delta=True, final_observation=True)
    h, d = make_env("walk", n, auto_reset=True, **kw), make_env("walk", n, auto_reset=True, **kw)
    plain = make_env("walk", n, auto_reset=False, **kw)
    assert int(h._L.rexsim_host_final_bytes(h._h)) == h._h_final.numel() == n * h.obs_dim * 4 + n
    np.testing.assert_array_equal(h.reset(), d.reset())
    plain.reset()
    rng = np.random.default_rng(1)
    ended = 0
    for k in range(16):
        a = rng.uniform(-1, 1, size=(n, 2)).astype(np.float32)
        oh, rh, dh, _ = h.step(a)
        od, rd, dd, _ = d.step(torch.from_numpy(a).cuda())
        np.testing.assert_array_equal(oh, _np(od), err_msg=f"obs {k}")
        np.testing.assert_array_equal(rh, _np(rd)); np.testing.assert_array_equal(dh, _np(dd))
        ended += dh.sum()
        np.testing.assert_array_equal(h.final_observation(), _np(d.final_observation()), err_msg=f"final {k}")
        np.testing.assert_array_equal(h.limit_bytes(), _np(d.limit_bytes()), err_msg=f"limit {k}")
        op, _, dp, _ = plain.step(a)
        np.testing.assert_array_equal(plain.final_observation()[dp], op[dp])
        if dp.any():
            plain.reset(np.nonzero(dp)[0])
        if k == 9:
            dev = torch.tensor([2, -1, n + 3], dtype=torch.int32, device="cuda")
            fin = h.final_observation().copy()
            d.reset(dev); h.reset(dev)
            for e in (h, d):
                with pytest.raises(IndexError):
                    e.check_errors()
            np.testing.assert_array_equal(h.final_observation(), fin)
    assert ended >= n
    h.close(); d.close(); plain.close()


# ---- GPU: rollouts ---------------------------------------------------------------------------------------------------------
def _rollout_env_net(kind, n):
    from rex_gym_b200.agents import ForwardGaussianPolicy, RecurrentGaussianPolicy
    from twin import make_env
    kw = dict(signal_type="ik", normalize=True, auto_reset=True, max_episode_steps=11, target_position=2.0, backwards=False, seed=6)
    env = make_env("walk", n, **kw)
    if kind == "ff":
        net = ForwardGaussianPolicy(env.obs_dim, env.action_dim, seed=3)
    else:
        net = RecurrentGaussianPolicy(env.obs_dim, env.action_dim, seed=3, num_envs=n)
    return env, net, kw


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ff", "gru"])
def test_graph_rollout_equals_the_loop_and_a_replay(kind):
    """Rollout(final_observation=True) captured as one graph equals the step-by-step loop bit for bit over two collects (every
    buffer, final_observ and truncated included); its final rows and truncation flags are what step_into writes on a replay
    of the recorded actions.  With the switch off a collect launches what it launched before: T step kernels."""
    import torch
    from rex_gym_b200.agents import Rollout
    from twin import make_env
    n, T = 256, 16
    outs = []
    for use_graph in (False, True):
        env, net, kw = _rollout_env_net(kind, n)
        ro = Rollout(env, net, T, seed=17, training=True, use_graph=use_graph, final_observation=True)
        a = {k: v.clone() for k, v in ro.collect().items()}
        b = {k: v.clone() for k, v in ro.collect().items()}
        assert {"final_observ", "truncated"} <= set(a)
        outs.append((a, b))
        if use_graph:
            hand = make_env("walk", n, **kw)
            obs = torch.zeros((n, env.obs_dim), device="cuda")
            r, d = torch.zeros(n, device="cuda"), torch.zeros(n, dtype=torch.uint8, device="cuda")
            fin, lim = torch.zeros_like(obs), torch.zeros(n, dtype=torch.uint8, device="cuda")
            hand.reset(torch.arange(n, dtype=torch.int32, device="cuda"))
            for rec in (a, b):
                for t in range(T):
                    hand.step_into(rec["action"][t].contiguous(), obs, r, d, fin, lim)
                    dt = _np(d).astype(bool)
                    np.testing.assert_array_equal(_np(rec["done"][t]), dt)
                    np.testing.assert_array_equal(_np(rec["final_observ"][t])[dt], _np(fin)[dt], err_msg=f"final {t}")
                    np.testing.assert_array_equal(_np(rec["truncated"][t]), _np(lim) == 1, err_msg=f"truncated {t}")
            hand.close()
        env.close(); net.close()
    (a0, b0), (a1, b1) = outs
    for k in a0:
        np.testing.assert_array_equal(_np(a0[k]), _np(a1[k]), err_msg=k)
        np.testing.assert_array_equal(_np(b0[k]), _np(b1[k]), err_msg=k)
    assert _np(b0["truncated"]).any()
    env, net, _ = _rollout_env_net(kind, n)
    ro = Rollout(env, net, T, seed=17, training=True, use_graph=False)
    assert "final_observ" not in ro.collect() and ro.final_observ is None
    before = env.launch_count, net.launch_count
    ro.collect()
    assert env.launch_count - before[0] == T
    assert net.launch_count - before[1] == (2 * T + 1 if kind == "ff" else 3 * T + 1)
    env.close(); net.close()


# ---- GPU: the bootstrap scan ----------------------------------------------------------------------------------------------
SCAN_LENGTHS = [1, 7, 8, 9, 1000]       # the scan loads 8 steps ahead: below, at and above 8, and far above


@pytest.mark.gpu
@pytest.mark.parametrize("T", SCAN_LENGTHS)
def test_bootstrap_scan_matches_the_fp64_restatement(T):
    """Every done / truncated pattern (truncated without done is ignored) at every unroll boundary, against the fp64
    restatement; with truncated all zero, bit-identical to gae_segments."""
    import torch
    from rex_gym_b200.agents import utility
    rng = np.random.default_rng(T)
    n = 300
    r = rng.normal(size=(T, n)).astype(np.float32)
    v = rng.normal(size=(T + 1, n)).astype(np.float32)
    fv = rng.normal(size=(T, n)).astype(np.float32)
    pattern = rng.integers(0, 4, size=(T, n))
    pattern[:, :4] = np.arange(4)[None, :]                  # columns 0..3: one pattern at every step
    d, tr = (pattern & 1) != 0, (pattern & 2) != 0
    c = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    for g, lam in ((0.985, 0.95), (0.9, 1.0)):
        ret, adv = utility.gae_segments(c(r), c(v), c(d), g, lam, truncated=c(tr), final_value=c(fv))
        wr, wa = gae_bootstrap_fp64(r, v, d, tr, fv, g, lam)
        np.testing.assert_allclose(_np(ret), wr, rtol=1e-5, atol=2e-5 * max(1, T / 100))
        np.testing.assert_allclose(_np(adv), wa, rtol=1e-5, atol=2e-5 * max(1, T / 100))
        cut = d & tr
        np.testing.assert_allclose(_np(adv)[cut], (r.astype(np.float64) + g * fv.astype(np.float64) - v[:T])[cut], atol=1e-5)
        zr, za = utility.gae_segments(c(r), c(v), c(d), g, lam, truncated=c(np.zeros_like(tr)), final_value=c(fv))
        pr, pa = utility.gae_segments(c(r), c(v), c(d), g, lam)
        np.testing.assert_array_equal(_np(zr), _np(pr)); np.testing.assert_array_equal(_np(za), _np(pa))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ff", "gru"])
def test_returns_bootstrap_from_the_oracle_value_of_final_observations(kind):
    """returns_and_advantages(bootstrap_truncated=True) after a graph collect: the fp64 restatement fed with the oracle network's
    value of the final observations of the truncated steps; without it, the plain scan; the cell state is untouched."""
    from rex_gym_b200.agents import Rollout
    n, T = 256, 24
    env, net, _ = _rollout_env_net(kind, n)
    ro = Rollout(env, net, T, seed=5, training=True, final_observation=True)
    ro.collect()
    out = {k: _np(v).copy() for k, v in ro.collect().items()}
    tr = out["truncated"]
    assert tr.any() and (tr <= out["done"]).all()
    hidden = _np(net._state).copy() if kind == "gru" else None
    ret, adv = ro.returns_and_advantages(0.985, 0.95, bootstrap_truncated=True)
    if hidden is not None:
        np.testing.assert_array_equal(_np(net._state), hidden)
    w, g = net.get_weights(), net.get_filters()
    f = AO.StreamingNormalize((env.obs_dim,), True, True, 5)
    f.count, f.mean, f.var_sum = g["observ_count"], g["observ_mean"].astype(np.float64), g["observ_var_sum"].astype(np.float64)
    fv = np.zeros((T, n))
    fv[tr] = _oracle_value(w, f, out["final_observ"][tr])
    wr, wa = gae_bootstrap_fp64(out["reward"], out["value"], out["done"], tr, fv, 0.985, 0.95)
    np.testing.assert_allclose(_np(ret), wr, rtol=1e-4, atol=2e-4)
    np.testing.assert_allclose(_np(adv), wa, rtol=1e-4, atol=2e-4)
    pr, pa = ro.returns_and_advantages(0.985, 0.95)
    wr0, wa0 = AO.gae_segments(out["reward"], out["value"], out["done"], 0.985, 0.95)
    np.testing.assert_allclose(_np(pr), wr0, rtol=1e-4, atol=2e-4)
    assert (np.abs(_np(ret) - _np(pr))[tr] > 1e-4).all()          # the bootstrap changed every truncated step
    env.close(); net.close()


def _oracle_value(w, f, observ):
    """The value network alone in fp64 (agent_oracle.forward_gaussian_policy's value half) on filtered observations."""
    x = f.transform(observ)
    W = {k: np.asarray(w[k], np.float64) for k in ("vW1", "vb1", "vW2", "vb2", "vW3", "vb3")}
    h = np.maximum(x @ W["vW1"] + W["vb1"], 0)
    h = np.maximum(h @ W["vW2"] + W["vb2"], 0)
    return (h @ W["vW3"] + W["vb3"])[:, 0]
