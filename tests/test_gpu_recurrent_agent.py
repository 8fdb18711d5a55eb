"""GPU: RecurrentGaussianPolicy and LinearGaussianPolicy (csrc/rexsim_agent.cu gru_policy_kernel / linear_policy_kernel, C ABI
include/rexsim_recurrent.h) against the fp64 oracle (oracle/recurrent_oracle.py), bit for bit where the kernels promise it,
and through Rollout.

gru_policy_kernel runs 64-env tiles on min(tiles, SMs) persistent CTAs; the value network is perform_kernel on the value block
with up to one CTA per SM (128-env tiles once there are as many as SMs).  The batch sizes sit on both sides of each switch.

Error bound: every pre-activation of the cell is an fp32 dot product of K = H1 + G <= 384 terms (300 for the shipped sizes)
whose absolute values sum to about 11 with these weights; sequential fp32 accumulation is off by at most K * 2^-24 * 11 = 2e-4,
and sigmoid / tanh do not amplify it.  So the new state, the mean and the sampled action are held to 2e-4, the log-prob to
2e-4 (as the feed-forward tests) and the value, which is the feed-forward kernel's, to 5e-5.  The cell is contractive (u < 1),
so the state error must not grow along the sequence: at step 64 it stays within 4x its value at step 8 (or 2^-20)."""
import numpy as np
import pytest
import torch

from agent_twin import (GRU_ROWS, LIN_ROWS, OFFSET, SEED, fitted_filter, ff_value_twin, gru_batch_sizes, gru_id, gru_net,
                        gru_weights, lin_id, lin_net, lin_weights, load, noise, observations, sampled, sm_count, tile_probes,
                        to_numpy)
from oracle import recurrent_oracle as RO

pytestmark = pytest.mark.gpu

TOL = dict(hidden=2e-4, mean=2e-4, action=2e-4, logprob=2e-4, value=5e-5)


@pytest.mark.parametrize("row", GRU_ROWS, ids=gru_id)
def test_perform_matches_the_oracle_over_a_sequence(row):
    """64 control steps with fresh observations and random episode starts (5 % of the rows per step) at every batch size: the
    mean, sampled action, log-prob, value and new state of probe rows against the oracle; the value is bit-identical to the
    feed-forward network's with the same value weights."""
    O, A, H1, G, vl = row
    rng = np.random.default_rng(100 * O + 10 * A + H1 + G)
    w, f = gru_weights(rng, O, A, H1, G, vl), fitted_filter(rng, O)
    sizes = gru_batch_sizes()
    N = max(sizes)
    net, ff = gru_net(row, N, w, f), ff_value_twin(O, A, vl, w, f)
    worst = {k: 0.0 for k in TOL}
    for n in sizes:
        net.load_state_dict(dict(net.state_dict(), hidden=torch.zeros_like(net.state_dict()["hidden"])))
        idx = tile_probes(n)
        h = np.zeros((len(idx), G))
        err_h = []
        for t in range(64):
            obs = observations(rng, n, O, outliers=0.01)                     # clipped after normalisation
            begin = rng.random(n) < 0.05
            x, b = torch.from_numpy(obs).cuda(), torch.from_numpy(begin.astype(np.uint8)).cuda()
            g = to_numpy(net.perform(x, training=True, seed=SEED, step=t, env_offset=OFFSET, begin=b))
            hid = net.state_dict()["hidden"][torch.from_numpy(idx).cuda()].cpu().numpy()
            _, mean, _, value, h = RO.perform(w, f, obs[idx], False, state=h, begin=begin[idx])
            action, logprob = sampled(mean, w["logstd"], noise(SEED, t, OFFSET + idx, A))
            e = dict(hidden=np.abs(hid - h).max(), mean=np.abs(g["mean"][idx] - mean).max(),
                     action=np.abs(g["action"][idx] - action).max(), value=np.abs(g["value"][idx] - value).max(),
                     logprob=np.abs(g["logprob"][idx] - logprob).max())
            for k in TOL:
                assert e[k] < TOL[k], (n, t, k, e[k])
                worst[k] = max(worst[k], e[k])
            err_h.append(e["hidden"])
            if t in (0, 63):
                assert np.array_equal(to_numpy(ff.perform(x, training=False))["value"], g["value"]), (n, t)
        assert max(err_h[56:]) <= 4 * max(max(err_h[:8]), 2.0 ** -20), (n, err_h[:8], err_h[56:])
    print("worst errors", gru_id(row), worst)
    net.close(); ff.close()


def _snapshot(row, n, steps=3, seed=5):
    """A network after `steps` steps with random begins, its state S, and the next step's inputs."""
    O, A, H1, G, vl = row
    rng = np.random.default_rng(seed)
    w, f = gru_weights(rng, O, A, H1, G, vl), fitted_filter(rng, O)
    net = gru_net(row, n, w, f)
    for t in range(steps):
        x = torch.from_numpy(rng.normal(0.3, 3.0, (n, O)).astype(np.float32)).cuda()
        net.perform(x, training=True, seed=SEED, step=t, env_offset=OFFSET,
                    begin=torch.from_numpy((rng.random(n) < 0.2).astype(np.uint8)).cuda())
    x = torch.from_numpy(rng.normal(0.3, 3.0, (n, O)).astype(np.float32)).cuda()
    m = torch.from_numpy((rng.random(n) < 0.3).astype(np.uint8)).cuda()
    return net, w, f, net.state_dict(), x, m


def _run(net, sd, x, m, **kw):
    net.load_state_dict(sd)
    out = to_numpy(net.perform(x, begin=m, **kw))
    out["hidden"] = net.state_dict()["hidden"].cpu().numpy()
    return out


def _rows_of(sd, rows):
    return dict(filters=sd["filters"], counters=sd["counters"], hidden=sd["hidden"][rows].clone())


KEYS = ("action", "mean", "logprob", "value", "hidden")


@pytest.mark.parametrize("row", GRU_ROWS[:2] + GRU_ROWS[5:6], ids=gru_id)
def test_begin_continue_value_only_position_and_shards_bit_for_bit(row):
    n = 64 * sm_count() + 37                                           # several tiles on some CTAs
    net, w, f, S, x, m = _snapshot(row, n)
    kw = dict(training=True, seed=SEED, step=7, env_offset=OFFSET)
    ref = _run(net, S, x, m, **kw)
    mb = m.cpu().numpy().astype(bool)
    # a begin row equals a fresh network's output for the same observation
    fresh = gru_net(row, n, w, f)
    fr = to_numpy(fresh.perform(x, **kw))
    fr["hidden"] = fresh.state_dict()["hidden"].cpu().numpy()
    for k in KEYS:
        assert np.array_equal(ref[k][mb], fr[k][mb]), k
    # rows without begin continue their state: begin changes nothing else
    cont = _run(net, S, x, None, **kw)
    for k in KEYS:
        assert np.array_equal(ref[k][~mb], cont[k][~mb]), k
    assert not np.array_equal(ref["hidden"][mb], cont["hidden"][mb])
    # a value-only call leaves the state untouched
    net.load_state_dict(S)
    v = net.perform(x, training=False, out=dict(value=torch.full((n,), float("nan"), device="cuda")))["value"].cpu().numpy()
    assert np.array_equal(v, ref["value"]) and torch.equal(net.state_dict()["hidden"], S["hidden"])
    # a row's outputs do not depend on its position in the batch (noise-free: the keys move with the position)
    det = _run(net, S, x, m, training=False)
    perm = torch.from_numpy(np.random.default_rng(2).permutation(n)).cuda()
    sp = _rows_of(S, perm)
    pd = _run(net, sp, x[perm].contiguous(), m[perm].contiguous(), training=False)
    p = perm.cpu().numpy()
    for k in ("mean", "value", "hidden"):
        assert np.array_equal(pd[k], det[k][p]), k
    # a shard (env_offset = k) reproduces the rows of the whole batch, sampling included; so does a lone env
    for k0, k1 in ((37, n), (0, 1), (n - 1, n), (64, 129)):
        shard = gru_net(row, k1 - k0, w, f)
        out = _run(shard, _rows_of(S, slice(k0, k1)), x[k0:k1].contiguous(), m[k0:k1].contiguous(), training=True, seed=SEED,
                   step=7, env_offset=OFFSET + k0)
        for k in KEYS:
            assert np.array_equal(out[k], ref[k][k0:k1]), (k0, k1, k)
        shard.close()
    fresh.close(); net.close()


def test_sampling_noise_is_the_feed_forward_networks():
    """With zero mean heads both networks sample action = exp(logstd) * eps exactly: the recurrent, linear and feed-forward
    networks draw the same eps for the same (seed, env_offset + env, step), and give the same log-prob."""
    O, A, H1, G, vl = GRU_ROWS[1]
    rng = np.random.default_rng(3)
    w, f = gru_weights(rng, O, A, H1, G, vl), fitted_filter(rng, O)
    w.update(pW3=np.zeros((G, A), np.float32), pb3=np.zeros(A, np.float32))
    n = 5000
    net = gru_net(GRU_ROWS[1], n, w, f)
    ff = ff_value_twin(O, A, vl, w, f, dict(pW3=np.zeros((vl[1], A), np.float32), pb3=np.zeros(A, np.float32), logstd=w["logstd"]))
    lin = lin_net(O, A, vl, n, dict(w, pW=np.zeros((O, A), np.float32), pb=np.zeros(A, np.float32)), f)
    x = torch.from_numpy(rng.normal(size=(n, O)).astype(np.float32)).cuda()
    kw = dict(training=True, seed=SEED, step=11, env_offset=OFFSET)
    a, b, c = to_numpy(net.perform(x, **kw)), to_numpy(ff.perform(x, **kw)), to_numpy(lin.perform(x, **kw))
    for k in ("action", "logprob", "value"):
        assert np.array_equal(a[k], b[k]) and np.array_equal(c[k], b[k]), k
    assert np.abs(a["action"]).max() > 0.1
    net.close(); ff.close(); lin.close()


@pytest.mark.parametrize("row", LIN_ROWS, ids=lin_id)
def test_linear_policy_matches_the_oracle(row):
    O, A, vl = row
    rng = np.random.default_rng(7 * O + A)
    f = fitted_filter(rng, O)
    w = lin_weights(rng, O, A, vl)
    sizes = [1, 127, 128, 129, 65536 + 37]
    net = lin_net(O, A, vl, max(sizes), w, f)
    obs = observations(rng, max(sizes), O)
    for n in sizes:
        g = to_numpy(net.perform(torch.from_numpy(obs[:n]).cuda(), training=True, seed=SEED, step=3, env_offset=OFFSET))
        idx = tile_probes(n, 128)
        _, want_m, _, want_v, _ = RO.perform(w, f, obs[idx], False)
        want_a, want_lp = sampled(want_m, w["logstd"], noise(SEED, 3, OFFSET + idx, A))
        assert np.abs(g["mean"][idx] - want_m).max() < 2e-5 and np.abs(g["value"][idx] - want_v).max() < TOL["value"], n
        assert np.abs(g["action"][idx] - want_a).max() < 5e-5 and np.abs(g["logprob"][idx] - want_lp).max() < TOL["logprob"], n
    net.close()


# ---- Rollout --------------------------------------------------------------------------------------------------------------
ENV_KW = dict(task="walk", signal_type="ik", normalize=True, auto_reset=True, max_episode_steps=10, target_position=2.0,
              backwards=False, control_latency=0.02, pd_latency=0.003)


def _rollout(cls, n, T, use_graph, training, **netkw):
    import rex_gym_b200 as R
    from rex_gym_b200.agents import Rollout
    env = R.BatchedRexEnv(num_envs=n, **ENV_KW)
    net = cls(env.obs_dim, env.action_dim, seed=3, num_envs=n, **netkw)
    return env, net, Rollout(env, net, T, seed=17, training=training, use_graph=use_graph)


def _replay(w, f, windows, G):
    """The oracle through the recorded observations and done flags of consecutive collects: begin is all ones at the first
    step, then the previous step's done."""
    n = windows[0]["observ"].shape[1]
    h, begin, out = np.zeros((n, G)), np.ones(n, bool), []
    for win in windows:
        for t in range(win["observ"].shape[0]):
            _, mean, _, value, h = RO.perform(w, f, win["observ"][t], False, state=h, begin=begin)
            out.append((mean, value))
            begin = win["done"][t].astype(bool)
    return out, h


def test_recurrent_rollout_graph_loop_oracle_and_resume():
    """walk-ik with auto_reset, latency and observation noise: the captured graph equals the step-by-step loop bit for bit
    (training, two collects); a host replay of the recorded observations and done flags through the oracle matches the
    deterministic rollout's means, values and final state within the sequence bound, across envs that restart mid-rollout;
    state_dict / load_state_dict resumes a collect bit for bit."""
    from rex_gym_b200.agents import RecurrentGaussianPolicy
    n, T = 512, 16
    outs = []
    for use_graph in (False, True):
        env, net, ro = _rollout(RecurrentGaussianPolicy, n, T, use_graph, True)
        a = {k: v.clone() for k, v in ro.collect().items()}
        b = {k: v.clone() for k, v in ro.collect().items()}
        outs.append((a, b, net.state_dict()["hidden"].clone()))
        env.close(); net.close()
    (a0, b0, h0), (a1, b1, h1) = outs
    for k in a0:
        assert torch.equal(a0[k], a1[k]) and torch.equal(b0[k], b1[k]), k
    assert torch.equal(h0, h1) and a0["done"].any() and b0["done"].any()

    env, net, ro = _rollout(RecurrentGaussianPolicy, n, T, True, False)
    rng = np.random.default_rng(4)
    w = net.get_weights()
    w.update(w_ru=(w["w_ru"] * 2).astype(np.float32), b_ru=rng.normal(0, 1, w["b_ru"].shape).astype(np.float32))
    f = fitted_filter(rng, env.obs_dim)
    load(net, w, f)
    wins = [{k: v.clone().cpu().numpy() for k, v in ro.collect().items()} for _ in range(2)]
    want, h = _replay(w, f, wins, net.G)
    got = [(win["mean"][t], win["value"][t]) for win in wins for t in range(T)]
    em = max(np.abs(g[0] - o[0]).max() for g, o in zip(got, want))
    ev = max(np.abs(g[1] - o[1]).max() for g, o in zip(got, want))
    eh = np.abs(net.state_dict()["hidden"].cpu().numpy() - h).max()
    assert em < TOL["mean"] and ev < TOL["value"] and eh < TOL["hidden"], (em, ev, eh)
    restarted = wins[0]["done"][:-1].any(0)
    assert restarted.sum() > 0
    # resume: put env, network and the rollout's carried observation and episode starts back, collect again
    snap = (env.state_dict(), net.state_dict(), ro._cur.clone(), ro._begin.clone())
    first = {k: v.clone() for k, v in ro.collect().items()}
    h_first = net.state_dict()["hidden"].clone()
    env.load_state_dict(snap[0]); net.load_state_dict(snap[1]); ro._cur.copy_(snap[2]); ro._begin.copy_(snap[3])
    again = ro.collect()
    for k in first:
        assert torch.equal(first[k], again[k]), k
    assert torch.equal(net.state_dict()["hidden"], h_first)
    env.close(); net.close()


def test_linear_rollout_runs_and_matches_the_oracle():
    from rex_gym_b200.agents import LinearGaussianPolicy
    n, T = 512, 16
    env, net, ro = _rollout(LinearGaussianPolicy, n, T, True, False)
    rng = np.random.default_rng(6)
    f = fitted_filter(rng, env.obs_dim)
    load(net, f=f)
    w = net.get_weights()
    win = {k: v.clone().cpu().numpy() for k, v in ro.collect().items()}
    for t in range(T):
        _, mean, _, value, _ = RO.perform(w, f, win["observ"][t], False)
        assert np.abs(win["mean"][t] - mean).max() < 2e-5 and np.abs(win["value"][t] - value).max() < TOL["value"], t
    assert np.array_equal(win["action"], win["mean"]) and win["done"].any()
    env.close(); net.close()
