"""CPU: the fp64 restatement of RecurrentGaussianPolicy / LinearGaussianPolicy (oracle/recurrent_oracle.py) against the
GRUBlockCell definition element by element and by hand, why torch.nn.GRUCell is not that cell, and the C ABI of
include/rexsim_recurrent.h: its export list, its parameter block sizes and the acceptance rule of rexrnn_create (rexrnn_check,
which create runs before its first CUDA call)."""
import ctypes as C
import math
import os
import re

import numpy as np
import torch

from oracle import recurrent_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, ERR_INVALID, ERR_UNSUPPORTED = 0, -1, -4
GRU, LINEAR = 0, 1


def _cell_by_element(x, h, w_ru, b_ru, w_c, b_c):
    """GRUBlockCell written out per unit from the TF 1.15 op documentation."""
    n, I = x.shape
    G = h.shape[1]
    out = np.zeros((n, G))
    for e in range(n):
        xh = list(x[e]) + list(h[e])
        r = [1 / (1 + math.exp(-(b_ru[j] + sum(xh[k] * w_ru[k, j] for k in range(I + G))))) for j in range(G)]
        u = [1 / (1 + math.exp(-(b_ru[G + j] + sum(xh[k] * w_ru[k, G + j] for k in range(I + G))))) for j in range(G)]
        xrh = list(x[e]) + [r[j] * h[e, j] for j in range(G)]
        for j in range(G):
            c = math.tanh(b_c[j] + sum(xrh[k] * w_c[k, j] for k in range(I + G)))
            out[e, j] = u[j] * h[e, j] + (1 - u[j]) * c
    return out


def _random_cell(rng, I, G):
    return (rng.normal(0, 0.5, (I + G, 2 * G)), 1.0 + rng.normal(0, 0.2, 2 * G), rng.normal(0, 0.5, (I + G, G)),
            rng.normal(0, 0.2, G))


def test_gru_block_cell_equals_the_op_documentation_per_element():
    rng = np.random.default_rng(0)
    for I, G in ((1, 1), (3, 4), (6, 5)):
        x, h = rng.normal(size=(4, I)), rng.uniform(-1, 1, (4, G))
        w = _random_cell(rng, I, G)
        np.testing.assert_allclose(RO.gru_block_cell(x, h, *w), _cell_by_element(x, h, *w), rtol=0, atol=1e-13)


def test_gru_block_cell_one_unit_by_hand():
    """x = h = 1, w_ru = 0, b_ru = (0, ln 3): r = 1/2, u = 3/4; w_c = (1, 2), b_c = 0: c = tanh(1 + 2 * 1/2) = tanh 2;
    h' = 3/4 * 1 + 1/4 * tanh 2.  Swapping r and u would give tanh(2.5) in c and 1/2 as the blend."""
    got = RO.gru_block_cell(np.ones((1, 1)), np.ones((1, 1)), np.zeros((2, 2)), np.array([0.0, math.log(3.0)]),
                            np.array([[1.0], [2.0]]), np.zeros(1))
    assert abs(got[0, 0] - (0.75 + 0.25 * math.tanh(2.0))) < 1e-15


def _torch_gru_cell(x, h, w_ru, b_ru, w_c, b_c):
    """torch.nn.GRUCell loaded with the same numbers: gates r, z from the same columns, n = tanh(W_in x + b_in + r * (W_hn h))."""
    I, G = x.shape[1], h.shape[1]
    cell = torch.nn.GRUCell(I, G).double()
    with torch.no_grad():
        cell.weight_ih.copy_(torch.from_numpy(np.concatenate([w_ru[:I].T, w_c[:I].T])))
        cell.weight_hh.copy_(torch.from_numpy(np.concatenate([w_ru[I:].T, w_c[I:].T])))
        cell.bias_ih.copy_(torch.from_numpy(np.concatenate([b_ru, b_c])))
        cell.bias_hh.zero_()
        return cell(torch.from_numpy(x), torch.from_numpy(h)).numpy()


def test_torch_gru_cell_is_a_different_cell():
    """torch applies r after the hidden matmul (r * (W h)) where GRUBlockCell applies it before (W (r * h)).  With one unit the
    two coincide; with two they do not, so torch.nn.GRUCell cannot check this cell."""
    rng = np.random.default_rng(1)
    x, h = rng.normal(size=(3, 2)), rng.uniform(-1, 1, (3, 1))
    w = _random_cell(rng, 2, 1)
    np.testing.assert_allclose(_torch_gru_cell(x, h, *w), RO.gru_block_cell(x, h, *w), rtol=0, atol=1e-14)
    h2 = rng.uniform(-1, 1, (3, 2))
    w2 = _random_cell(rng, 2, 2)
    assert np.abs(_torch_gru_cell(x, h2, *w2) - RO.gru_block_cell(x, h2, *w2)).max() > 1e-2


def test_recurrent_abi_exports_every_declared_symbol():
    from rex_gym_b200 import _capi
    L = _capi.load()
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rexsim_recurrent.h")).read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(rexrnn_[a-z0-9_]+)\s*\(", src)))
    assert len(names) == 9 and sorted(_capi.RNN_EXPORTS) == names
    for n in names:
        assert hasattr(L, n), n


def _cfgs(O, A, H1v, H2v, kind, H1, G, num_envs=1):
    from rex_gym_b200 import _capi
    return _capi.RexAgentConfig(O, A, H1v, H2v, 5.0, 10.0), _capi.RexRnnConfig(kind, H1, G, num_envs)


def test_parameter_block_sizes_match_the_oracle_packing():
    from rex_gym_b200 import _capi
    L = _capi.load()
    for O, A, H1, G in ((4, 2, 200, 100), (16, 4, 200, 100), (1, 1, 4, 4), (32, 8, 256, 128), (4, 3, 36, 8)):
        for kind, shapes in ((GRU, RO.gru_shapes(O, A, H1, G)), (LINEAR, RO.linear_shapes(O, A))):
            a, r = _cfgs(O, A, 200, 100, kind, H1, G)
            w = {k: np.arange(np.prod(s), dtype=np.float32).reshape(s) + i for i, (k, s) in enumerate(shapes)}
            block = RO.pack_policy(w, shapes)
            assert L.rexrnn_policy_floats(C.byref(a), C.byref(r)) == block.size and block.size % 4 == 0
            back = RO.unpack_policy(block, shapes)
            for k, _ in shapes:
                np.testing.assert_array_equal(back[k], w[k])
    a, r = _cfgs(4, 2, 200, 100, GRU, 200, 100)
    # 800 + 200 + 300 * 200 + 200 + 300 * 100 + 100 + 200 + 2 + 2 = 91 504: the 90 000 cell weights dominate
    assert L.rexrnn_policy_floats(C.byref(a), C.byref(r)) == 91504


def test_create_refuses_exactly_past_each_limit():
    from rex_gym_b200 import _capi
    L = _capi.load()
    cases = [  # (O, A, kind, hidden1, cell, num_envs), the code rexrnn_check returns
        ((1, 1, GRU, 4, 4, 1), OK), ((32, 8, GRU, 256, 128, 1), OK), ((4, 2, GRU, 200, 100, 65536), OK),
        ((0, 2, GRU, 200, 100, 1), ERR_INVALID), ((33, 2, GRU, 200, 100, 1), ERR_INVALID),
        ((4, 0, GRU, 200, 100, 1), ERR_INVALID), ((4, 9, GRU, 200, 100, 1), ERR_INVALID),
        ((4, 2, GRU, 0, 100, 1), ERR_UNSUPPORTED), ((4, 2, GRU, 260, 100, 1), ERR_UNSUPPORTED),
        ((4, 2, GRU, 202, 100, 1), ERR_UNSUPPORTED), ((4, 2, GRU, 200, 0, 1), ERR_UNSUPPORTED),
        ((4, 2, GRU, 200, 132, 1), ERR_UNSUPPORTED), ((4, 2, GRU, 200, 102, 1), ERR_UNSUPPORTED),
        ((4, 2, GRU, 200, 100, 0), ERR_INVALID), ((4, 2, 2, 200, 100, 1), ERR_INVALID), ((4, 2, -1, 200, 100, 1), ERR_INVALID),
        ((4, 2, LINEAR, 0, 0, 1), OK), ((32, 8, LINEAR, 999, 999, 1), OK), ((33, 2, LINEAR, 0, 0, 1), ERR_INVALID),
        ((4, 2, LINEAR, 0, 0, 0), ERR_INVALID),
    ]
    for (O, A, kind, H1, G, n), want in cases:
        a, r = _cfgs(O, A, 64, 12, kind, H1, G, n)
        assert L.rexrnn_check(C.byref(a), C.byref(r)) == want, ((O, A, kind, H1, G, n), want)
    a, r = _cfgs(4, 2, 64, 14, GRU, 200, 100)                # the agent's own rule first: hidden2 not a multiple of 4
    assert L.rexrnn_check(C.byref(a), C.byref(r)) == ERR_UNSUPPORTED
    h = C.c_void_p()
    assert L.rexrnn_create(None, C.byref(r), C.byref(h)) == ERR_INVALID
