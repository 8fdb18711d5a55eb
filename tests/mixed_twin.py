"""A batch that mixes per-env constructor keywords, checked against one scalar-built twin per group of envs: the bitwise row and
state comparisons and a twin runner keyed on a group label.

Not collected by pytest (like twin.py): the tests import what they need from here.
"""
import numpy as np

from twin import LAYOUT, bound, make_env


def bits(t):
    """A tensor with its float32 words as int32, so that == compares bit for bit (NaNs and signed zeros included)."""
    import torch
    t = torch.as_tensor(t).contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def assert_rows_equal(a, b, rows, what):
    """Rows `rows` of a and b (tensors or arrays, env-major) equal bit for bit."""
    import torch
    rows = torch.as_tensor(rows, device=torch.as_tensor(a).device).long()
    if rows.numel() == 0:
        return
    a, b = bits(a), bits(b)
    bad = (a[rows] != b[rows]).reshape(len(rows), -1).any(1)
    assert not bad.any(), "%s differs in envs %s" % (what, rows.cpu()[bad.cpu()].tolist())


def assert_envs_equal(mixed, twin, envs, what):
    """Every raw state word (float and int, by name from the kernel's header) of `envs`, bit for bit, and the envs' columns
    of the sensor history ring."""
    import torch
    sel = torch.as_tensor(np.asarray(envs), device="cuda").long()
    f1, f2 = mixed._state_f[:, sel], twin._state_f[:, sel]
    i1, i2 = mixed._state_i[:, sel], twin._state_i[:, sel]
    for w in range(LAYOUT.NF):
        assert torch.equal(bits(f1[w]), bits(f2[w])), "%s: float word %d of envs %s" % (what, w, list(envs))
    for w in range(LAYOUT.NI):
        assert torch.equal(i1[w], i2[w]), "%s: int word %d of envs %s" % (what, w, list(envs))
    assert (mixed._ring is None) == (twin._ring is None)
    if mixed._ring is not None:
        n = mixed.num_envs
        assert torch.equal(bits(mixed._ring.view(-1, n)[:, sel]), bits(twin._ring.view(-1, n)[:, sel])), "%s: ring" % what


def label_groups(labels):
    """{label: env indices} of a per-env label list, labels in order of first appearance."""
    labels = list(labels)
    return {g: np.array([e for e, l in enumerate(labels) if l == g]) for g in dict.fromkeys(labels)}


def run_twins(task, n, mixed_kw, twin_kw, labels, steps=36, reset_at=17, rebalance_at=9, extra=None):
    """A mixed batch of n envs (make_env(task, n, auto_reset=True, **mixed_kw)) and one twin per group label
    (make_env(task, n, auto_reset=True, **twin_kw[label])), stepped on the same actions with auto-reset, one explicit reset
    whose indices span every group, and a re-grouping (rexsim_rebalance) mid-run: every env's outputs and state words equal
    its group's twin's, bit for bit.  extra(mixed, twin, envs, step) adds checks after each step.
    -> (mixed, {label: twin}, {label: env indices})."""
    import torch
    groups = label_groups(labels)
    mixed = make_env(task, n, auto_reset=True, **mixed_kw)
    twins = {g: make_env(task, n, auto_reset=True, **twin_kw[g]) for g in groups}
    everyone = torch.arange(n, dtype=torch.int32, device="cuda")
    o = mixed.reset(everyone)
    for g, tw in twins.items():
        assert_rows_equal(o, tw.reset(everyone), groups[g], "reset obs, %s" % (g,))
        assert_envs_equal(mixed, tw, groups[g], "after reset, %s" % (g,))
    gen = torch.Generator(device="cuda"); gen.manual_seed(3)
    b = bound(task, mixed_kw.get("signal_type", "ik"))
    mid = torch.tensor(sorted({int(e[len(e) // 2]) for e in groups.values()} | {n - 1}), dtype=torch.int32, device="cuda")
    for k in range(steps):
        if k == rebalance_at:
            mixed._call(mixed._L.rexsim_rebalance, mixed._h)       # slots re-sorted within each group's range
        a = (torch.rand((n, mixed.action_dim), device="cuda", generator=gen) * 2 - 1) * b
        om, rm, dm, _ = mixed.step(a)
        om, rm, dm = om.clone(), rm.clone(), dm.clone()
        for g, tw in twins.items():
            ot, rt, dt, _ = tw.step(a)
            assert_rows_equal(om, ot, groups[g], "obs, step %d, %s" % (k, g))
            assert_rows_equal(rm, rt, groups[g], "reward, step %d, %s" % (k, g))
            assert_rows_equal(dm, dt, groups[g], "done, step %d, %s" % (k, g))
            assert_envs_equal(mixed, tw, groups[g], "step %d, %s" % (k, g))
            if extra:
                extra(mixed, tw, groups[g], k)
        if k == reset_at:
            r = mixed.reset(mid)
            for g, tw in twins.items():
                sel = np.nonzero(np.isin(mid.cpu().numpy(), groups[g]))[0]
                assert_rows_equal(r, tw.reset(mid), sel, "explicit reset obs, %s" % (g,))
    assert mixed.check_errors() == 0
    return mixed, twins, groups
