"""perform (csrc/rexsim_agent.cu) restated in numpy in the kernels' own fp32 arithmetic.

Not collected by pytest (like task_outputs.py).  The restatement follows the kernel source, not the TF graph:

* the normaliser of load_normaliser / filter_inv_std and load_obs_tile, in float32 operations;
* layer 1 as both kernels compute it: b1[k], then one fmaf per input o = 0 .. O-1, then the ReLU;
* perform_kernel<TM> (fp32): layer 2 as acc = b2, then one fmaf per k = 0 .. H1-1; head part 1 per group of 4 columns
  fmaf(r0, w3[0], fmaf(r1, w3[1], fmaf(r2, w3[2], r3 * w3[3]))); head part 2 b3 plus the groups in order.  Every operation
  is in an order fixed by the code, so the head sums (the value, and the argument of the mean's tanhf) come out bit for bit;
* perform_tc_kernel<O, A> (tf32): layer 2's operands rounded with cvt.rna.tf32.f32, then D_n = sum_k a_k b_kn and
  S_n = sum_k |a_k b_kn| in fp64 (the products are exact there, and fp64 summation error is about 2^-30 of the accumulation
  model below, so it is negligible); the head in fp64 from D with a forward error bound for every output;
* gru_policy_kernel and linear_policy_kernel: every GEMM of the cell, the blend and both heads are fmaf chains in an order
  the code fixes (fma_chain; the cp.async chunking of gru_gemm does not reorder the rows), so what reaches sigmoidf / tanhf
  comes out bit for bit; sigmoidf, tanhf and the sampler (head_outputs) are held to error bounds built from the library's
  documented maximum ulp errors.

fmaf32 is a correctly rounded fp32 fused multiply-add, vectorised; the tests check it against the C library's fmaf.
"""
import math

import numpy as np

F32 = np.float32
U32 = 2.0 ** -24                  # unit roundoff of fp32
OBSERV_CLIP, REWARD_CLIP = 5.0, 10.0          # the clips ForwardGaussianPolicy configures (algorithm.py:49-58)
# CUDA's tanhf: at most 2 ulp from the exact tanh over the whole range (CUDA C++ Programming Guide, maximum ulp errors of
# the single-precision mathematical functions); the library is built without fast-math, so this is the tanhf that runs
TANHF_ULP = 2
# the same table for the other functions the agent kernels call; sqrtf and fp32 division are correctly rounded (0 ulp) in a
# build without fast-math (nvcc's -prec-sqrt and -prec-div default to true)
EXPF_ULP, LOGF_ULP, COSPIF_ULP = 2, 1, 1
# sigmoidf(x) = 1 / (1 + expf(-x)) is exactly 1 for x >= SIGMOID_ONE (expf(-24) < 2^-25 even with expf's error, so 1 + E
# rounds to 1) and exactly 0 for x <= SIGMOID_ZERO (expf(96) overflows to inf); tests/test_gpu_recurrent_rounding.py asserts both
SIGMOID_ONE, SIGMOID_ZERO = 24.0, -96.0
FLT_MAX = float(np.finfo(F32).max)
LOGPROB_C = F32(0.9189385332046727)           # head_outputs' 0.5 log(2 pi), as the fp32 constant the kernel uses


# ---- fp32 arithmetic --------------------------------------------------------------------------------------------------
def fmaf32(a, b, c):
    """Correctly rounded float32 a * b + c.  The product of two float32 values is exact in fp64; c is added in fp64 with
    TwoSum giving the rounding error of that addition; the fp64 sum is then rounded to float32.  That second rounding is
    only wrong where the fp64 sum lies exactly on a float32 midpoint while the exact sum does not: there the sign of the
    TwoSum error decides the direction."""
    a, b, c = np.broadcast_arrays(np.asarray(a, F32), np.asarray(b, F32), np.asarray(c, F32))
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bv = s - p
    err = (p - (s - bv)) + (c64 - bv)                      # p + c == s + err exactly
    r = s.astype(F32)
    r64 = r.astype(np.float64)
    other = np.where(r64 > s, np.nextafter(r, F32(-np.inf)), np.nextafter(r, F32(np.inf)))
    tie = (r64 != s) & ((r64 + other.astype(np.float64)) * 0.5 == s) & (err != 0)
    return np.where(tie, np.where(err > 0, np.maximum(r, other), np.minimum(r, other)), r)


def tf32_rna(x):
    """cvt.rna.tf32.f32: add 0x1000 to the bit pattern and clear the low 13 bits -- ties away from zero, a carry into the
    exponent where the mantissa rounds up into the next binade, the sign kept."""
    u = np.ascontiguousarray(x, F32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(F32)


def ulp32(t):
    """The spacing of float32 numbers at |t| (t in fp64): 2^(e - 24) for 2^(e-1) <= |t| < 2^e, at least 2^-149."""
    _, e = np.frexp(np.abs(np.asarray(t, np.float64)))
    return np.ldexp(1.0, np.maximum(e - 24, -149))


def within_tanhf(mean, z):
    """|mean - tanh(z)| in units of tanhf's error bound (<= 1 passes); z: the exact argument, in fp64."""
    t = np.tanh(np.asarray(z, np.float64))
    return np.abs(np.asarray(mean, np.float64) - t) / (TANHF_ULP * ulp32(t))


# ---- exactness of a constructed network -------------------------------------------------------------------------------
def _mantissa(x):
    """|x| = N * 2^(e - 53) with N a 53-bit integer, and the trailing zero bits of N (x in fp64, zeros dropped)."""
    x = np.abs(np.asarray(x, np.float64)).ravel()
    x = x[x != 0]
    m, e = np.frexp(x)
    N = np.ldexp(m, 53).astype(np.int64)
    tz = np.frexp((N & -N).astype(np.float64))[1] - 1
    return e, tz


def significant_bits(x):
    """Largest number of significant bits of any element (0 for an all-zero array)."""
    _, tz = _mantissa(x)
    return int((53 - tz).max()) if tz.size else 0


def grid_exponent(x):
    """Smallest m with every element an integer multiple of 2^-m."""
    e, tz = _mantissa(x)
    return int((53 - e - tz).max()) if tz.size else -1074


def assert_exact_dot(x, W, b, what):
    """Every partial sum of b + x @ W, in any order and grouping, is exact in fp32: all terms lie on the grid 2^-m and
    sum |terms| * 2^m < 2^24 for every dot product.  Returns the exact result (fp64)."""
    x, W, b = (np.asarray(v, np.float64) for v in (x, W, b))
    m = max(grid_exponent(x) + grid_exponent(W), grid_exponent(b))
    total = np.abs(x) @ np.abs(W) + np.abs(b)
    assert float(np.ldexp(total.max(), m)) < 2.0 ** 24, (what, m, float(total.max()))
    return x @ W + b


# ---- the normaliser and layer 1 (both kernels) ----------------------------------------------------------------------
def normaliser(count, mean, var_sum):
    """load_normaliser: the means and 1 / (sqrt(var_sum / (count - 1) + 1e-4) + 1e-8) in float32, exactly 1 while
    count <= 1."""
    mean, vs = np.asarray(mean, F32), np.asarray(var_sum, F32)
    if count > 1:
        inv = F32(1) / (np.sqrt(vs / F32(count - 1) + F32(1e-4)) + F32(1e-8))
    else:
        inv = np.ones_like(vs)
    return mean, inv.astype(F32)


def normalise(obs, mean, inv, clip=OBSERV_CLIP):
    """load_obs_tile: (v - mean) * inv, then the clip, in float32."""
    v = (np.asarray(obs, F32) - mean) * inv
    return np.minimum(np.maximum(v, F32(-clip)), F32(clip))


def transform_reward(r, count, var_sum, clip=REWARD_CLIP):
    """transform_reward_kernel: fminf(fmaxf(r * inv, -clip), clip) in float32."""
    _, inv = normaliser(count, np.zeros(1), np.asarray([var_sum]))
    return np.minimum(np.maximum(np.asarray(r, F32) * inv[0], F32(-clip)), F32(clip))


def layer1(x, W1, b1):
    """relu(b1[k] + fmaf over o = 0 .. O-1) as float32 [R][H1]."""
    x, W1 = np.asarray(x, F32), np.asarray(W1, F32)
    s = np.broadcast_to(np.asarray(b1, F32), (x.shape[0], W1.shape[1]))
    for o in range(x.shape[1]):
        s = fmaf32(x[:, o:o + 1], W1[o][None, :], s)
    return np.maximum(s, F32(0))


def net_params(w, net):
    """(W1, b1, W2, b2, W3, b3) of the policy (net 0) or the value network (net 1) as float32."""
    p = "pv"[net]
    return tuple(np.asarray(w[p + k], F32) for k in ("W1", "b1", "W2", "b2", "W3", "b3"))


# ---- perform_kernel<TM> ---------------------------------------------------------------------------------------------------
def head_sums_fp32(x, W1, b1, W2, b2, W3, b3):
    """perform_kernel's head sums s (b3 included), float32 [R][AO]: the value (AO = 1) or the arguments of tanhf."""
    h1 = layer1(x, W1, b1)
    R, H2 = h1.shape[0], W2.shape[1]
    acc = np.broadcast_to(b2, (R, H2))
    for k in range(h1.shape[1]):
        acc = fmaf32(h1[:, k:k + 1], W2[k][None, :], acc)
    r = np.maximum(acc, F32(0)).reshape(R, H2 // 4, 4, 1)
    w3 = W3.reshape(1, H2 // 4, 4, -1)
    part = fmaf32(r[:, :, 0], w3[:, :, 0], fmaf32(r[:, :, 1], w3[:, :, 1], fmaf32(r[:, :, 2], w3[:, :, 2], r[:, :, 3] * w3[:, :, 3])))
    s = np.broadcast_to(b3, (R, W3.shape[1])).astype(F32)
    for g in range(H2 // 4):
        s = s + part[:, g]
    return s


# ---- perform_tc_kernel<O, A> --------------------------------------------------------------------------------------------
def layer2_tf32(h1, W2):
    """D = a @ b and S = |a| @ |b| in fp64, a = tf32_rna(h1) [R][H1] and b = tf32_rna(W2) [H1][H2]."""
    a, b = tf32_rna(h1).astype(np.float64), tf32_rna(W2).astype(np.float64)
    return a @ b, np.abs(a) @ np.abs(b)


def accumulation_bound(S, H1):
    """The tensor cores' accumulation model: every product exact, one rounding (truncation allowed) per m64n16k8 step,
    so |d - D| <= (ceil(H1 / 8) + 1) * 2^-23 * S."""
    return (math.ceil(H1 / 8) + 1) * 2.0 ** -23 * S


def head_tf32(D, S, b2, W3, b3, H1):
    """The epilogue and head in fp64 from D, with a forward error bound per output: (z, bound), [R][AO] each.

    d within the accumulation model of D; then fp32 d + b2 (one rounding) and the ReLU (1-Lipschitz); the head's fp32 sum
    of H2 products and b3 rounds at most 4 * ceil(H2 / 16) + 3 times on any path (a fmaf per column in each lane's chain,
    two shuffle additions, b3), bounded by gamma_k times the sum of the absolute terms."""
    b2, W3, b3 = (np.asarray(v, np.float64) for v in (b2, W3, b3))
    E = accumulation_bound(S, H1)
    pre = D + b2
    H = np.maximum(pre, 0)
    eh = E + U32 * (np.abs(pre) + E)
    k = 4 * (-(-W3.shape[0] // 16)) + 3
    gamma = k * U32 / (1 - k * U32)
    aW3 = np.abs(W3)
    bound = eh @ aW3 + gamma * ((H + eh) @ aW3 + np.abs(b3))
    return H @ W3 + b3, bound


def tanh_bound(z, bz):
    """Bound on |tanhf(z') - tanh(z)| for |z' - z| <= bz: the largest slope of tanh on that interval times bz, plus
    tanhf's own error."""
    z = np.asarray(z, np.float64)
    t = np.tanh(z)
    return bz / np.cosh(np.maximum(np.abs(z) - bz, 0)) ** 2 + TANHF_ULP * ulp32(np.abs(t) + bz)


# ---- the transcendental functions and their bounds -------------------------------------------------------------------------
def sigmoid_bound(x):
    """Bound on |sigmoidf(x) - sigmoid(x)| for float32 x: expf's error on E = exp(-x), the rounding of 1 + E, its effect on
    1 / D (|1/D' - 1/D| <= |D' - D| / (D (D - |D' - D|))) and the correctly rounded division.  Where expf(-x) may overflow to
    inf in fp32, sigmoidf gives 0 and sigmoid(x) itself is added."""
    x = np.asarray(x, np.float64)
    with np.errstate(over="ignore"):
        E = np.exp(-x)
    E = np.minimum(E, 2.0 ** 200)                          # beyond fp32's range the formula only needs to stay finite
    dE = EXPF_ULP * ulp32(E)
    D = 1.0 + E
    dD = dE + 0.5 * ulp32(D + dE)
    s = 1.0 / D
    di = dD / (D * (D - dD))
    return di + 0.5 * ulp32(s + di) + np.where(E * (1 + 2.0 ** -21) >= FLT_MAX, s, 0.0)


def sigmoid(x):
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-np.asarray(x, np.float64)))


def uniforms(r):
    """head_outputs' uniform of a 32-bit draw r: ((float)(r >> 9) + 0.5f) * 2^-23, in float32 operations."""
    k = (np.asarray(r, np.uint64) >> np.uint64(9)).astype(F32)
    return (k + F32(0.5)) * F32(2.0 ** -23)


def normal_bound(u1, u2):
    """z = sqrtf(-2 logf(u1)) * cospif(2 u2) for float32 u1, u2 (exact): the exact z and a bound on the kernel's error.
    logf within LOGF_ULP; -2 logf and 2 u2 are exact scalings; sqrtf correctly rounded; cospif within COSPIF_ULP; the
    product rounded once."""
    u1, u2 = np.asarray(u1, np.float64), np.asarray(u2, np.float64)
    L = np.log(u1)
    dT = 2 * LOGF_ULP * ulp32(L)
    T = -2.0 * L
    S = np.sqrt(T)
    dS = dT / (np.sqrt(np.maximum(T - dT, 0.0)) + S)
    dS = dS + 0.5 * ulp32(S + dS)
    Cs = np.cos(2.0 * np.pi * u2)
    dC = COSPIF_ULP * ulp32(Cs)
    Z = S * Cs
    dZ = S * dC + np.abs(Cs) * dS + dS * dC
    return Z, dZ + 0.5 * ulp32(np.abs(Z) + dZ)


def action_bound(z, dz, logstd, mean):
    """act = fmaf(expf(ls), z', mu) against mean + exp(ls) z: (the exact value, bound); mean is the kernel's own mu."""
    E = np.exp(np.asarray(logstd, np.float64))
    dE = EXPF_ULP * ulp32(E)
    act = np.asarray(mean, np.float64) + E * z
    d = E * dz + np.abs(z) * dE + dE * dz
    return act, d + 0.5 * ulp32(np.abs(act) + d)


def logprob_bound(z, dz, logstd):
    """lp = sum over a of -0.5f * z * z - ls - c (c = LOGPROB_C) against the same sum of the exact z, in fp64: (value, bound).
    The bound covers the code as written and every FMA contraction nvcc may apply under its default --fmad=true: each of
    the at most 4 A roundings (the product by z, the two subtractions, the accumulation) is at most u times the largest
    intermediate, which is below M = sum (0.5 (|z| + dz)^2 + |ls| + c); a contraction only removes roundings.  z's own
    error enters through |z'^2 - z^2| / 2 <= dz (2 |z| + dz) / 2."""
    z, dz = np.asarray(z, np.float64), np.asarray(dz, np.float64)
    ls = np.asarray(logstd, np.float64)
    c = float(LOGPROB_C)
    lp = (-0.5 * z * z - ls - c).sum(-1)
    M = (0.5 * (np.abs(z) + dz) ** 2 + np.abs(ls) + c).sum(-1)
    k = 4 * z.shape[-1]
    return lp, (dz * (2 * np.abs(z) + dz) / 2).sum(-1) + k * U32 / (1 - k * U32) * M


# ---- gru_policy_kernel / linear_policy_kernel ------------------------------------------------------------------------------
def fma_chain(x, W, b):
    """b[j], then one fmaf(x[:, k], W[k, j], .) per row k = 0 .. K-1 in order: float32 [R][C].  This is gru_gemm (x = [a1, h]
    or [a1, r h], rows below H1 from a1; the 16-row chunks are consumed in order, each from its first row), the GRU head
    (x = h', W = W3, b = b3), the linear policy (x = the normalised observation, W = pW, b = pb) and layer1 before the ReLU."""
    x, W = np.asarray(x, F32), np.asarray(W, F32)
    acc = np.broadcast_to(np.asarray(b, F32), (x.shape[0], W.shape[1]))
    for k in range(W.shape[0]):
        acc = fmaf32(x[:, k:k + 1], W[k][None, :], acc)
    return acc


def gru_blend(u, h, t):
    """h' = fmaf(u, h, (1 - u) * t) with t = tanhf(c): 1 - u and the product each rounded in fp32."""
    u, h, t = (np.asarray(v, F32) for v in (u, h, t))
    return fmaf32(u, h, (F32(1) - u) * t)


def gru_gate_sums(a1, h, w):
    """The pre-activations [r | u] of the cell, bit for bit: b_ru, then the rows of w_ru over [a1, h] in order."""
    return fma_chain(np.concatenate([a1, h], 1), w["w_ru"], w["b_ru"])


def chain_bound(x, dx, W, b):
    """Two fmaf chains over the same W and b, the reference on float32 inputs x, the other on inputs within dx of them:
    (the reference's float32 result, a bound on the distance of the two).  Per row k the bound grows by |W[k]| dx[k] and,
    once the two chains differ, by half an ulp of each chain's partial sum.  Identical inputs into identical partial
    sums give identical results, so the bound stays 0 until the first row with dx > 0."""
    x, W = np.asarray(x, F32), np.asarray(W, F32)
    dx = np.asarray(dx, np.float64)
    aW = np.abs(W.astype(np.float64))
    acc = np.broadcast_to(np.asarray(b, F32), (x.shape[0], W.shape[1]))
    e = np.zeros(acc.shape)
    for k in range(W.shape[0]):
        acc = fmaf32(x[:, k:k + 1], W[k][None, :], acc)
        grow = e + dx[:, k:k + 1] * aW[k][None, :]
        a = np.abs(acc.astype(np.float64))
        e = np.where(grow > 0, grow + 0.5 * ulp32(a + ulp32(a) + grow) + 0.5 * ulp32(a), 0.0)
    return acc, e


def gru_step_bound(w, a1, h):
    """One step of gru_policy_kernel from its dense activations a1 and state h (float32, begin rows already zero), against
    the GRU cell applied to the kernel's own gate sums: (h' reference, bound, head sums s, bound on s).

    The gate sums are the kernel's bit for bit (gru_gate_sums).  From there: r and u within sigmoid_bound of sigmoid;
    r h rounded once, so |rh - F32(sigmoid(r) h)| <= sb_r |h| + half an ulp of each; the candidate chain over [a1, rh]
    within chain_bound of the reference chain over F32(sigmoid(r) h); tanhf within tanh_bound; then 1 - u (one
    rounding), the product (one rounding) and the fmaf blend (one rounding) each add their operands' bounds times the
    other operand and half an ulp.  h' is compared with u h + (1 - u) tanh(c) in fp64 (c: the reference chain).  The head
    is chain_bound over F32(h'), its inputs within the bound on h' plus that rounding; the mean is then within
    tanh_bound(s, bound on s) of tanh(s)."""
    a1, h = np.asarray(a1, F32), np.asarray(h, F32)
    G = h.shape[1]
    pre = gru_gate_sums(a1, h, w).astype(np.float64)
    r, u = sigmoid(pre[:, :G]), sigmoid(pre[:, G:])
    sb = sigmoid_bound(pre)
    sr, su = sb[:, :G], sb[:, G:]
    h64 = h.astype(np.float64)
    rh_ex = r * h64
    rh = rh_ex.astype(F32)
    drh = sr * np.abs(h64) + 0.5 * ulp32(np.abs(rh_ex) + sr * np.abs(h64)) + np.abs(rh.astype(np.float64) - rh_ex)
    dx = np.concatenate([np.zeros(a1.shape), drh], 1)
    c, ec = chain_bound(np.concatenate([a1, rh], 1), dx, w["w_c"], w["b_c"])
    c = c.astype(np.float64)
    t, dt = np.tanh(c), tanh_bound(c, ec)
    om = 1.0 - u
    dom = su + 0.5 * ulp32(om + su)
    q = om * t
    dq = dom * np.abs(t) + om * dt + dom * dt
    dq = dq + 0.5 * ulp32(np.abs(q) + dq)
    hp = u * h64 + q
    dh = su * np.abs(h64) + dq
    dh = dh + 0.5 * ulp32(np.abs(hp) + dh)
    h32 = hp.astype(F32)
    s, es = chain_bound(h32, dh + np.abs(h32.astype(np.float64) - hp), w["pW3"], w["pb3"])
    return hp, dh, s, es
