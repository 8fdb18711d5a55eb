// rexsim_agent.cu -- device-side agent glue around the step kernel (include/rexsim_agent.h):
//   perform     : StreamingNormalize.transform + ForwardGaussianPolicy (policy MLP, value MLP) + sampling, one fused kernel
//   rexrnn_*    : the RecurrentGaussianPolicy (GRU) and LinearGaussianPolicy policies of include/rexsim_recurrent.h
//   experience  : StreamingNormalize.update for observations and rewards, one deterministic reduction kernel
//   scans       : discounted_return / lambda_advantage (reference row semantics) and the done-aware time-major GAE
// fp32 throughout (the reference's TF graph is fp32): the MLP is computed on the CUDA cores with a register-tiled
// shared-memory GEMM so results match an fp32 reference to rounding; see DESIGN.md for the roofline of each kernel.
#include "rexsim_kernel.cuh"
#include "rexsim_host.h"
#include "../../include/rexsim_agent.h"
#include "../../include/rexsim_recurrent.h"
#include <cstring>
#include <vector>
#include <type_traits>

namespace rexsim {

constexpr int AG_MAX_O = 32, AG_MAX_A = 8, AG_MAX_H1 = 256, AG_MAX_H2 = 128;
constexpr int RED_BLOCKS = 256;    // partial blocks of the filter update

struct AgentDev {
    RexAgentConfig cfg;
    const float* __restrict__ params;    // policy block | value block
    int pol_floats, val_floats;
    float* filt;                          // observ mean[O], var_sum[O], reward mean, var_sum
    int64_t* cnt;                         // observ count, reward count, step counter, blocks-done ticket
                                          // (64-bit: at 65 536 envs a 32-bit count wraps after 32 768 control steps)
    float* partial;                       // [RED_BLOCKS][2 * (O + 1)]
};

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }

// One network's packed parameter block (include/rexsim_agent.h), offsets in floats: W1 [O][H1], b1 [H1], W2 [H1][H2], b2 [H2],
// W3 [H2][AO], b3 [AO], then the policy's logstd [A]; AO = A for the policy, 1 for the value network; padded to 4 floats.
// I: the index type of the caller's address arithmetic -- int64_t in perform_kernel and the exported sizes, int in
// perform_tc_kernel (the type that keeps each kernel's registers and instruction count at or below the hand-chained form).
template <typename I> struct ParamLayout { I W1, b1, W2, b2, W3, b3, logstd, floats; };
template <typename I>
__host__ __device__ constexpr ParamLayout<I> param_layout(I O, I A, I H1, I H2, bool policy) {
    const I AO = policy ? A : 1, b1 = O * H1, W2 = b1 + H1, b2 = W2 + H1 * H2, W3 = b2 + H2, b3 = W3 + H2 * AO, ls = b3 + AO;
    return {0, b1, W2, b2, W3, b3, ls, (ls + (policy ? A : 0) + 3) & ~(I)3};
}

// filt = [observ mean O | observ var_sum O | reward mean | reward var_sum]: column j < O is observation j, column O the reward
__device__ __forceinline__ float* filt_mean(float* filt, int O, int col) { return col < O ? &filt[col] : &filt[2 * O]; }
__device__ __forceinline__ float* filt_var_sum(float* filt, int O, int col) { return col < O ? &filt[O + col] : &filt[2 * O + 1]; }
// StreamingNormalize's 1 / (std + 1e-8), std = sqrt(var_sum / (count - 1) + 1e-4) (normalize.py:57-66, _std :131-144); 1 until
// the count passes 1
__device__ __forceinline__ float filter_inv_std(float var_sum, int64_t count) {
    float inv = 1.f;
    if (count > 1) inv = 1.f / (sqrtf(var_sum / (float)(count - 1) + 1e-4f) + 1e-8f);
    return inv;
}
// after a filter update over n rows: both counts advance by n, the step counter by one (the next perform draws fresh noise)
__device__ __forceinline__ void advance_counts(const AgentDev& D, int64_t n) { D.cnt[0] += n; D.cnt[1] += n; D.cnt[2] += 1; }

struct PerformArgs {
    AgentDev D;
    const float* __restrict__ observ;
    int n, training;
    int net_base;                         // perform_kernel: network of blockIdx.y = 0 (1: the value network alone)
    uint64_t seed;
    uint32_t step, env_offset;
    float* action; float* mean; float* logprob; float* value; float* observ_copy;
};

// StreamingNormalize.transform constants of the O observation columns -> nrm = [mean O | 1 / (std + 1e-8) O]
__device__ __forceinline__ void load_normaliser(const AgentDev& D, int O, float* nrm, int tid) {
    if (tid < O) {
        const int64_t cnt = D.cnt[0];
        const float m = *filt_mean(D.filt, O, tid), vs = *filt_var_sum(D.filt, O, tid);
        nrm[tid] = m; nrm[O + tid] = filter_inv_std(vs, cnt);
    }
}

// normalised, clipped observations of the TM-env tile starting at env e0 -> xs [O][TM] (zeros past n), threads tid, tid + nt, ..
// reading the [TM][O] block coalesced; the policy CTAs (net 0) copy the raw rows to observ_copy on the way
template <int TM>
__device__ __forceinline__ void load_obs_tile(const PerformArgs& P, int O, int net, const float* nrm, float* xs, int e0, int tid,
                                              int nt) {
    for (int i = tid; i < TM * O; i += nt) {
        const int e = i / O, o = i - e * O;
        float v = 0.f;
        if (e0 + e < P.n) {
            v = P.observ[(size_t)(e0 + e) * O + o];
            if (net == 0 && P.observ_copy) P.observ_copy[(size_t)(e0 + e) * O + o] = v;
        }
        v = (v - nrm[o]) * nrm[O + o];
        v = fminf(fmaxf(v, -P.D.cfg.observ_clip), P.D.cfg.observ_clip);
        xs[o * TM + e] = v;
    }
}

// one env's outputs from its head sums s (b3 included): the value (net 1), or per action tanh -> mean, the sample of
// network.policy.sample (algorithm.py:116) when training, and the diag-normal log-density (net 0).  AC: the head width at
// compile time; 0 = the first A of s[AG_MAX_A].
template <int AC, int AU>
__device__ __forceinline__ void head_outputs(const PerformArgs& P, int net, int A, int env, uint32_t step, const float (&s)[AU],
                                             const float* logstd) {
    if (net == 1) {
        if (P.value) P.value[env] = s[0];
    } else {
        float lp = 0.f;
#pragma unroll
        for (int a = 0; a < AU; a++) {
            if (AC || a < A) {
                const float mu = tanhf(s[a]);
                const float ls = logstd[a];
                float act = mu, z = 0.f;
                if (P.training) {
                    // u = (k + 1/2) 2^-23 for the top 23 bits k: k + 0.5 has at most 24 significant bits, so u is exact in fp32
                    // and lies in [2^-24, 1 - 2^-24] (never 1, where logf would give z = 0)
                    const uint32_t genv = P.env_offset + (uint32_t)env;
                    const float u1 = ((float)(rand_u32(P.seed, genv, step, 2 * a) >> 9) + 0.5f) * 0x1p-23f;
                    const float u2 = ((float)(rand_u32(P.seed, genv, step, 2 * a + 1) >> 9) + 0.5f) * 0x1p-23f;
                    z = sqrtf(-2.f * logf(u1)) * cospif(2.f * u2);
                    act = fmaf(expf(ls), z, mu);
                }
                lp += -0.5f * z * z - ls - 0.9189385332046727f;
                if (P.action) P.action[(size_t)env * A + a] = act;
                if (P.mean) P.mean[(size_t)env * A + a] = mu;
            }
        }
        if (P.logprob) P.logprob[env] = lp;
    }
}

// dynamic shared memory of perform_kernel<TM>, offsets in floats after the weights of the larger network (wmax floats):
// xs [AG_MAX_O][TM], h1 [H1][TM] (reused for the head partials [H2/4][TM][AO]), nrm [2][AG_MAX_O]
struct PerformSmem { size_t xs, h1, nrm, bytes; };
__host__ __device__ constexpr PerformSmem perform_smem(int wmax, int H1, int tm) {
    const size_t xs = wmax, h1 = xs + (size_t)AG_MAX_O * tm, nrm = h1 + (size_t)H1 * tm;
    return {xs, h1, nrm, (nrm + 2 * AG_MAX_O) * sizeof(float)};
}

// Persistent CTAs, blockIdx.y = network (0 policy, 1 value): weights -> shared memory once (TMA bulk copy), then for every
// tile of TM envs:  normalise -> layer 1 (O x H1) -> layer 2 (H1 x H2: TM/16 envs x 4 outputs per thread, register tile) ->
// head (H2 x A | 1) from the register tile + a shared-memory reduction over the H2/4 column groups -> tanh / sampling.
// blockDim.x = 16 * (H2 / 4)  (400 threads for the reference's 200-100 networks).
template <int TM>
__global__ void __launch_bounds__(512, 1) perform_kernel(const PerformArgs P) {
    constexpr int RE = TM / 16;                           // envs per thread in the layer-2 register tile
    extern __shared__ __align__(16) float smem[];
    __shared__ __align__(8) uint64_t bar;
    const RexAgentConfig& c = P.D.cfg;
    const int O = c.obs_dim, A = c.action_dim, H1 = c.hidden1, H2 = c.hidden2;
    const int nt = blockDim.x, tid = threadIdx.x;
    const int net = blockIdx.y + P.net_base;
    const PerformSmem S = perform_smem(max(P.D.pol_floats, P.D.val_floats), H1, TM);
    float* W = smem;                          // weights of this CTA's network
    float* xs = smem + S.xs;
    float* h1 = smem + S.h1;
    float* nrm = smem + S.nrm;
    mbar_init(&bar);
    load_normaliser(P.D, O, nrm, tid);
    __syncthreads();
    const int ntiles = (P.n + TM - 1) / TM;
    const uint32_t step = P.step + (uint32_t)P.D.cnt[2];
    const int eg = tid & 15, og = tid >> 4;
    const int ngroups = H2 / 4;
    const bool l2_active = og < ngroups;              // the launch rounds the block up to TM threads for tiny networks
    const int AO = net == 0 ? A : 1;
    const int wfloats = net == 0 ? P.D.pol_floats : P.D.val_floats;
    // no proxy fence before the copy: nothing in this CTA has touched W through the generic proxy yet
    tma_bulk_load(W, P.D.params + (net == 0 ? 0 : P.D.pol_floats), (uint32_t)wfloats * 4u, &bar, 0u);
    const ParamLayout<int64_t> L = param_layout<int64_t>(O, A, H1, H2, net == 0);
    const float* W1 = W + L.W1; const float* b1 = W + L.b1;
    const float* W2 = W + L.W2; const float* b2 = W + L.b2;
    const float* W3 = W + L.W3; const float* b3 = W + L.b3;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int e0 = tile * TM;
        __syncthreads();                                // previous tile's head is done with h1
        load_obs_tile<TM>(P, O, net, nrm, xs, e0, tid, nt);
        __syncthreads();
        for (int i = tid; i < H1 * TM; i += nt) {       // layer 1
            const int k = i / TM, e = i - k * TM;
            float s = b1[k];
            for (int o = 0; o < O; o++) s = fmaf(xs[o * TM + e], W1[o * H1 + k], s);
            h1[i] = fmaxf(s, 0.f);
        }
        __syncthreads();
        // layer 2 register tile: acc[i][j] = env i of this thread x hidden unit 4*og + j; per k one LDS.128 of weights and
        // RE/4 LDS.128 of activations feed 4*RE FFMAs
        float acc[RE][4];
        if (l2_active) {
            const float4 bb = ld4(b2 + 4 * og);
#pragma unroll
            for (int i = 0; i < RE; i++) { acc[i][0] = bb.x; acc[i][1] = bb.y; acc[i][2] = bb.z; acc[i][3] = bb.w; }
            // thread's envs: chunk c (of RE/4) covers envs 64*c + 4*eg .. +3, so the 16 lanes of a half-warp read 256
            // contiguous bytes per LDS.128 (bank-conflict free; envs 8*eg .. 8*eg+7 would be a 4-way conflict)
            const float* hp = h1 + 4 * eg;
            const float* wp = W2 + 4 * og;
#pragma unroll 4
            for (int k = 0; k < H1; k++) {
                const float4 w = ld4(wp);
#pragma unroll
                for (int cidx = 0; cidx < RE / 4; cidx++) {
                    const float4 t = ld4(hp + cidx * 64);
                    const float hv[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
                    for (int l = 0; l < 4; l++) {
                        float* a = acc[4 * cidx + l];
                        a[0] = fmaf(hv[l], w.x, a[0]); a[1] = fmaf(hv[l], w.y, a[1]);
                        a[2] = fmaf(hv[l], w.z, a[2]); a[3] = fmaf(hv[l], w.w, a[3]);
                    }
                }
                hp += TM; wp += H2;
            }
        }
        __syncthreads();                                // all reads of h1 done: reuse it for the head partials
        if (l2_active) {                                // head, part 1: this thread's 4 hidden units x its RE envs
            float w3[4][AG_MAX_A];
#pragma unroll
            for (int j = 0; j < 4; j++)
#pragma unroll
                for (int a = 0; a < AG_MAX_A; a++) w3[j][a] = a < AO ? W3[(4 * og + j) * AO + a] : 0.f;
#pragma unroll
            for (int i = 0; i < RE; i++) {
                const float r0 = fmaxf(acc[i][0], 0.f), r1 = fmaxf(acc[i][1], 0.f), r2 = fmaxf(acc[i][2], 0.f), r3 = fmaxf(acc[i][3], 0.f);
                float* dst = h1 + ((size_t)og * TM + (i / 4) * 64 + 4 * eg + (i & 3)) * AO;
#pragma unroll
                for (int a = 0; a < AG_MAX_A; a++)
                    if (a < AO) dst[a] = fmaf(r0, w3[0][a], fmaf(r1, w3[1][a], fmaf(r2, w3[2][a], r3 * w3[3][a])));
            }
        }
        __syncthreads();
        if (tid < TM && e0 + tid < P.n) {               // head, part 2: one thread per env sums the column groups in order
            const int e = tid, env = e0 + e;
            float s[AG_MAX_A];
#pragma unroll
            for (int a = 0; a < AG_MAX_A; a++) s[a] = a < AO ? b3[a] : 0.f;
            for (int g = 0; g < ngroups; g++) {
                const float* src = h1 + ((size_t)g * TM + e) * AO;
#pragma unroll
                for (int a = 0; a < AG_MAX_A; a++) if (a < AO) s[a] += src[a];
            }
            head_outputs<0>(P, net, A, env, step, s, W + L.logstd);
        }
    }
}

// -------------------------------------------------------------------------------------------------------------------
// RecurrentGaussianPolicy / LinearGaussianPolicy policies (include/rexsim_recurrent.h).  The value network is the agent's
// perform_kernel on the value block alone (net_base = 1); normalisation, sampling and log-density are load_obs_tile and
// head_outputs above, so one (seed, env_offset + env, step) draws the same noise as ForwardGaussianPolicy.
// -------------------------------------------------------------------------------------------------------------------
constexpr int RNN_MAX_H1 = 256, RNN_MAX_G = 128;
constexpr int RNN_TM = 64;          // envs per tile: 4 per thread x 16 env groups
constexpr int RNN_KC = 16;          // weight rows per streamed chunk

// the GRU policy block (include/rexsim_recurrent.h), offsets in floats; every array starts on a 16-byte boundary (H1, G
// multiples of 4)
template <typename I> struct RnnLayout { I W1, b1, w_ru, b_ru, w_c, b_c, W3, b3, logstd, floats; };
template <typename I>
__host__ __device__ constexpr RnnLayout<I> rnn_layout(I O, I A, I H1, I G) {
    const I b1 = O * H1, wru = b1 + H1, bru = wru + (H1 + G) * 2 * G, wc = bru + 2 * G, bc = wc + (H1 + G) * G, W3 = bc + G,
            b3 = W3 + G * A, ls = b3 + A;
    return {0, b1, wru, bru, wc, bc, W3, b3, ls, (ls + A + 3) & ~(I)3};
}
// the linear policy block: W [O][A] at 0, b [A] at O * A, logstd [A] after it
__host__ __device__ constexpr int64_t linear_floats(int64_t O, int64_t A) { return (O * A + 2 * A + 3) & ~(int64_t)3; }

struct RnnArgs {
    PerformArgs P;                        // observations, filters, sampling keys, outputs (P.value is the value pass's)
    const float* __restrict__ params;     // the policy block
    float* state;                         // [num_envs][G]
    const uint8_t* __restrict__ begin;    // [n] or null
    int H1, G;
};

// dynamic shared memory of gru_policy_kernel, offsets in floats: xs [O][TM], a1 [H1][TM] (dense layer), h [G][TM] (state, then
// the new state), rh [G][TM] (r * h), w [2][KC][2G] (streamed weight chunks), head [TM][AG_MAX_A], nrm [2][AG_MAX_O]
struct RnnSmem { size_t xs, a1, h, rh, w, head, nrm, bytes; };
__host__ __device__ constexpr RnnSmem rnn_smem(int O, int H1, int G) {
    const size_t a1 = (size_t)O * RNN_TM, h = a1 + (size_t)H1 * RNN_TM, rh = h + (size_t)G * RNN_TM, w = rh + (size_t)G * RNN_TM,
                 head = w + 2 * (size_t)RNN_KC * 2 * G, nrm = head + (size_t)RNN_TM * AG_MAX_A;
    return {0, a1, h, rh, w, head, nrm, (nrm + 2 * AG_MAX_O) * sizeof(float)};
}

__device__ __forceinline__ void cp_async16(float* dst, const float* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }

// acc[s][i][j] += sum_k in[k][env 4 eg + i] * Wg[k][s G + 4 og + j] over the K = H1 + G rows of the cell input [x, hx]: rows
// k < H1 from a1, the rest from hx.  Wg [K][S G] is streamed from global memory (L2) in KC-row chunks through the two halves of
// wbuf, cp.async double-buffered: chunk c + 1 is in flight while chunk c is used.  Every thread calls this (it syncs); threads
// past the G / 4 column groups only help with the copies.  Per row: one LDS.128 of activations and S of weights feed 16 S FFMAs.
template <int S>
__device__ __forceinline__ void gru_gemm(const float* __restrict__ Wg, int H1, int G, const float* a1, const float* hx, float* wbuf,
                                         bool active, int eg, int og, int tid, int nt, float (&acc)[S][4][4]) {
    const int K = H1 + G, NC = S * G, nchunks = (K + RNN_KC - 1) / RNN_KC;
    const int half = RNN_KC * 2 * G;
    auto stage = [&](int c) {
        const int k0 = c * RNN_KC, rows = min(RNN_KC, K - k0);
        float* dst = wbuf + (c & 1) * half;
        const float* src = Wg + (size_t)k0 * NC;
        for (int i = 4 * tid; i < rows * NC; i += 4 * nt) cp_async16(dst + i, src + i);
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    stage(0);
    for (int c = 0; c < nchunks; c++) {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();                                // chunk c is in; every thread is done with chunk c - 1's half
        if (c + 1 < nchunks) stage(c + 1);
        if (!active) continue;
        const float* wb = wbuf + (c & 1) * half + 4 * og;
        const int k0 = c * RNN_KC, rows = min(RNN_KC, K - k0);
#pragma unroll 4
        for (int kk = 0; kk < rows; kk++) {
            const int k = k0 + kk;
            const float4 x = ld4((k < H1 ? a1 + (size_t)k * RNN_TM : hx + (size_t)(k - H1) * RNN_TM) + 4 * eg);
            const float xv[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
            for (int s = 0; s < S; s++) {
                const float4 w = ld4(wb + kk * NC + s * G);
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    acc[s][i][0] = fmaf(xv[i], w.x, acc[s][i][0]); acc[s][i][1] = fmaf(xv[i], w.y, acc[s][i][1]);
                    acc[s][i][2] = fmaf(xv[i], w.z, acc[s][i][2]); acc[s][i][3] = fmaf(xv[i], w.w, acc[s][i][3]);
                }
            }
        }
    }
}

// Persistent CTAs over 64-env tiles, one CTA per SM; per tile: normalise -> dense H1 ReLU -> gates [r | u] (register tile:
// 4 envs x 4 units of r and the same 4 units of u per thread) -> r * h -> candidate c (same tile) -> h' = u h + (1 - u) c in
// place of h -> state write-back -> head (one thread per (env, action)) -> tanh / sampling.  blockDim.x = max(16 G / 4, 128).
__global__ void __launch_bounds__(512, 1) gru_policy_kernel(const RnnArgs R) {
    const PerformArgs& P = R.P;
    extern __shared__ __align__(16) float smem[];
    const int O = P.D.cfg.obs_dim, A = P.D.cfg.action_dim, H1 = R.H1, G = R.G;
    const int nt = blockDim.x, tid = threadIdx.x, eg = tid & 15, og = tid >> 4;
    const bool active = og < G / 4;
    const RnnSmem S = rnn_smem(O, H1, G);
    float* xs = smem + S.xs; float* a1 = smem + S.a1; float* h = smem + S.h; float* rh = smem + S.rh;
    float* wbuf = smem + S.w; float* head = smem + S.head; float* nrm = smem + S.nrm;
    const RnnLayout<int64_t> L = rnn_layout<int64_t>(O, A, H1, G);
    const float* W = R.params;
    load_normaliser(P.D, O, nrm, tid);
    __syncthreads();
    const int ntiles = (P.n + RNN_TM - 1) / RNN_TM;
    const uint32_t step = P.step + (uint32_t)P.D.cnt[2];
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int e0 = tile * RNN_TM;
        __syncthreads();                                // previous tile's head is done with h and head
        load_obs_tile<RNN_TM>(P, O, 0, nrm, xs, e0, tid, nt);
        for (int i = tid; i < G * RNN_TM; i += nt) {    // the state rows, coalesced; zero where an episode begins and past n
            const int e = i / G, j = i - e * G, env = e0 + e;
            h[j * RNN_TM + e] = env < P.n && !(R.begin && R.begin[env]) ? R.state[(size_t)env * G + j] : 0.f;
        }
        __syncthreads();
        for (int i = tid; i < H1 * RNN_TM; i += nt) {   // dense layer
            const int k = i / RNN_TM, e = i - k * RNN_TM;
            float s = W[L.b1 + k];
            for (int o = 0; o < O; o++) s = fmaf(xs[o * RNN_TM + e], W[L.W1 + o * H1 + k], s);
            a1[i] = fmaxf(s, 0.f);
        }
        float ru[2][4][4], cc[1][4][4];
        if (active) {
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const float br = W[L.b_ru + 4 * og + j], bu = W[L.b_ru + G + 4 * og + j], bc = W[L.b_c + 4 * og + j];
#pragma unroll
                for (int i = 0; i < 4; i++) { ru[0][i][j] = br; ru[1][i][j] = bu; cc[0][i][j] = bc; }
            }
        }
        gru_gemm<2>(W + L.w_ru, H1, G, a1, h, wbuf, active, eg, og, tid, nt, ru);      // its first sync covers a1
        if (active) {                                   // r * h for the candidate; u stays in ru[1]
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int idx = (4 * og + j) * RNN_TM + 4 * eg + i;
                    rh[idx] = sigmoidf(ru[0][i][j]) * h[idx];
                    ru[1][i][j] = sigmoidf(ru[1][i][j]);
                }
        }
        __syncthreads();                                // rh complete; the weight halves are free again
        gru_gemm<1>(W + L.w_c, H1, G, a1, rh, wbuf, active, eg, og, tid, nt, cc);
        if (active) {                                   // nothing reads h any more but the thread that owns each element
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int idx = (4 * og + j) * RNN_TM + 4 * eg + i;
                    const float u = ru[1][i][j];
                    h[idx] = fmaf(u, h[idx], (1.f - u) * tanhf(cc[0][i][j]));
                }
        }
        __syncthreads();
        for (int i = tid; i < G * RNN_TM; i += nt) {    // the new state, coalesced
            const int e = i / G, j = i - e * G, env = e0 + e;
            if (env < P.n) R.state[(size_t)env * G + j] = h[j * RNN_TM + e];
        }
        for (int i = tid; i < RNN_TM * A; i += nt) {    // head sums, one thread per (env, action), b3 first then the units in order
            const int e = i / A, a = i - e * A;
            float s = W[L.b3 + a];
            for (int j = 0; j < G; j++) s = fmaf(h[j * RNN_TM + e], W[L.W3 + j * A + a], s);
            head[e * AG_MAX_A + a] = s;
        }
        __syncthreads();
        if (tid < RNN_TM && e0 + tid < P.n) {
            float s[AG_MAX_A];
#pragma unroll
            for (int a = 0; a < AG_MAX_A; a++) s[a] = a < A ? head[tid * AG_MAX_A + a] : 0.f;
            head_outputs<0>(P, 0, A, e0 + tid, step, s, W + L.logstd);
        }
    }
}

// LinearGaussianPolicy: one CTA per 128-env tile, one thread per env: s = b + x . W, then head_outputs
constexpr int LIN_TM = 128;
__global__ void __launch_bounds__(LIN_TM) linear_policy_kernel(const RnnArgs R) {
    const PerformArgs& P = R.P;
    __shared__ __align__(16) float xs[AG_MAX_O * LIN_TM];
    __shared__ float nrm[2 * AG_MAX_O];
    const int O = P.D.cfg.obs_dim, A = P.D.cfg.action_dim, tid = threadIdx.x, e0 = blockIdx.x * LIN_TM;
    const float* W = R.params;
    load_normaliser(P.D, O, nrm, tid);
    __syncthreads();
    load_obs_tile<LIN_TM>(P, O, 0, nrm, xs, e0, tid, LIN_TM);
    __syncthreads();
    if (e0 + tid >= P.n) return;
    float s[AG_MAX_A];
#pragma unroll
    for (int a = 0; a < AG_MAX_A; a++) {
        if (a < A) {
            float v = W[O * A + a];
            for (int o = 0; o < O; o++) v = fmaf(xs[o * LIN_TM + tid], W[o * A + a], v);
            s[a] = v;
        } else {
            s[a] = 0.f;
        }
    }
    head_outputs<0>(P, 0, A, e0 + tid, P.step + (uint32_t)P.D.cnt[2], s, W + O * A + A);
}


// -------------------------------------------------------------------------------------------------------------------
// perform on the tensor cores (opt-in: rexagent_set_precision(a, 1)).
//
// Layer 2 (H1 x H2 = 200 x 100, 97 % of the network's flops) runs as warpgroup MMAs (wgmma, sm_90a) per 128-env tile: each of
// the two warpgroups computes D[64 envs][NP] (fp32, registers) = A[64][H1] (layer-1 activations, shared memory) x B[NP][H1]^T
// (W2^T, shared memory) with m64n16k8 tf32 instructions (operands rounded to 10-bit mantissas with cvt.rna, fp32
// accumulation), NP = H2 rounded up to 16, H1 / 8 K-steps x NP / 16 column chunks issued asynchronously and waited for once.
// The epilogue reads the accumulators where wgmma leaves them (thread <-> two envs x pairs of columns), finishes bias, ReLU
// and the head per thread, sums the head over the four threads that share an env with two shuffles and samples one env per
// thread.  Layer 1 (O <= 16 inputs) and the head stay on the CUDA cores in fp32.
//
// Operand layout in shared memory: K-major, no swizzle (interleave): 8-row x 16-byte core matrices (8 rows x 4 tf32), the
// two core matrices one instruction reads along K are LBO bytes apart, 8-row groups SBO = 128 bytes apart:
//   byte(row, k) = (k / 4) * LBO + (row / 8) * 128 + (row % 8) * 16 + (k % 4) * 4,   LBO = rows * 16.
// Layer 1 writes A directly in that form (one 16-byte store per (env, 4 hidden units)).
// TF32 keeps 11 significant bits: tests/test_gpu_agent_rounding.py holds exact networks bit for bit and realistic ones to a
// bound propagated from the tensor cores' accumulation model; the fp32 kernel stays the parity default.
// -------------------------------------------------------------------------------------------------------------------
namespace tc {
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ float to_tf32(float x) { uint32_t r; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x)); return __uint_as_float(r); }
// wgmma shared-memory matrix descriptor: start address, leading / stride byte offsets (16-byte units), no swizzle,
// base offset 0
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((addr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
// D[64][16] (+)= A[64][8] x B[16][8]^T, both operands K-major in shared memory; accumulate = 0 overwrites D
__device__ __forceinline__ void wgmma_tf32_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %10, 0;\n"
                 " wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(da), "l"(db), "r"(accumulate) : "memory");
}
constexpr int TM = 128, THREADS = 256, NCH = AG_MAX_H2 / 16;    // two warpgroups x 64 envs; column chunks of 16
}  // namespace tc

static size_t perform_tc_smem_bytes(const RexAgentConfig* c) {
    const int npad = (c->hidden2 + 15) & ~15;
    const size_t a = (size_t)tc::TM * c->hidden1 * 4, b = (size_t)npad * c->hidden1 * 4;
    const size_t small = ((size_t)c->obs_dim * c->hidden1 + c->hidden1 + c->hidden2 + (size_t)c->hidden2 * AG_MAX_A + 2 * AG_MAX_A +
                          (size_t)c->obs_dim * tc::TM + 2 * AG_MAX_O) * 4;
    return a + b + small + 64;
}

// OT / AT: obs_dim / action_dim known at compile time (0 = generic: loops over the maxima with predicates -- every predicated-off
// instruction still takes an issue slot, which made the generic form 4x heavier than needed for the reference's 4-in / 2-out nets)
template <int OT, int AT>
__global__ void __launch_bounds__(tc::THREADS, 1) perform_tc_kernel(const PerformArgs P) {
    using namespace tc;
    extern __shared__ __align__(128) uint8_t smraw[];
    const RexAgentConfig& c = P.D.cfg;
    const int O = OT ? OT : c.obs_dim, A = AT ? AT : c.action_dim, H1 = c.hidden1, H2 = c.hidden2;
    constexpr int OU = OT ? OT : 16;                        // unroll bound of the input loops
    const int NP = (H2 + 15) & ~15;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int net = blockIdx.y;
    const int AO = net == 0 ? A : 1;
    const uint32_t LBO_A = TM * 16, LBO_B = (uint32_t)NP * 16;
    uint8_t* Asm = smraw;                                   // [H1/4][TM/8][8][16 B]
    uint8_t* Bsm = Asm + (size_t)TM * H1 * 4;               // [H1/4][NP/8][8][16 B]
    float* W1 = reinterpret_cast<float*>(Bsm + (size_t)NP * H1 * 4);   // [O][H1]
    float* b1 = W1 + O * H1;
    float* b2 = b1 + H1;
    float* W3 = b2 + H2;                                    // [H2][AO]
    float* b3 = W3 + H2 * AG_MAX_A;                         // b3[AO], then logstd[AO]
    float* xs = b3 + 2 * AG_MAX_A;                          // [O][TM]
    float* nrm = xs + O * TM;                               // [2][O]
    const float* G = P.D.params + (net == 0 ? 0 : P.D.pol_floats);
    const ParamLayout<int> L = param_layout(O, A, H1, H2, net == 0);
    const float* gW1 = G + L.W1; const float* gb1 = G + L.b1; const float* gW2 = G + L.W2; const float* gb2 = G + L.b2;
    const float* gW3 = G + L.W3; const float* gb3 = G + L.b3;
    load_normaliser(P.D, O, nrm, tid);
    // weights: the small layers as they are, W2 transposed into the B operand form (rounded to tf32, zero rows up to NP)
    for (int i = tid; i < O * H1; i += THREADS) W1[i] = gW1[i];
    for (int i = tid; i < H1; i += THREADS) b1[i] = gb1[i];
    for (int i = tid; i < H2; i += THREADS) b2[i] = gb2[i];
    for (int i = tid; i < H2 * AO; i += THREADS) W3[i] = gW3[i];
    if (tid < 2 * AO) b3[tid] = gb3[tid];                   // b3[AO] followed by logstd[AO] (policy block; unused for the value net)
    {   // W2 [H1][H2] row-major -> B[n][k]: 16-byte global loads (4 consecutive n of one k), several in flight per thread
        const int nq = NP >> 2;
#pragma unroll 4
        for (int i = tid; i < nq * H1; i += THREADS) {
            const int k = i / nq, n = (i - k * nq) << 2;
            float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
            if (n < H2) w = *reinterpret_cast<const float4*>(gW2 + (size_t)k * H2 + n);        // H2 is a multiple of 4
            uint8_t* dst = Bsm + (size_t)(k >> 2) * LBO_B + (n >> 3) * 128 + (n & 7) * 16 + (k & 3) * 4;
            *reinterpret_cast<float*>(dst) = to_tf32(w.x); *reinterpret_cast<float*>(dst + 16) = to_tf32(w.y);
            *reinterpret_cast<float*>(dst + 32) = to_tf32(w.z); *reinterpret_cast<float*>(dst + 48) = to_tf32(w.w);
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");         // B was written through the generic proxy
    __syncthreads();
    const int wg = warp >> 2;                               // warpgroup: tile rows 64 wg .. 64 wg + 63
    const int nch = NP >> 4;
    const uint32_t a_addr = smem_u32(Asm) + (uint32_t)wg * 1024u, b_addr = smem_u32(Bsm);
    const int ntiles = (P.n + TM - 1) / TM;
    const uint32_t step = P.step + (uint32_t)P.D.cnt[2];
    // a tile's observations -> xs: issued for the first tile here and for tile t + 1 right after the MMAs of tile t are issued,
    // so the global loads are in flight while the tensor cores run
    auto load_obs = [&](int tile) { load_obs_tile<TM>(P, O, net, nrm, xs, tile * TM, tid, THREADS); };
    if ((int)blockIdx.x < ntiles) load_obs(blockIdx.x);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int e0 = tile * TM;
        __syncthreads();
        // layer 1 -> A operand: thread = (env, half of the hidden units); the env's inputs stay in registers, the weight rows
        // are warp-wide broadcast loads, every 4 hidden units leave as one 16-byte store into the core-matrix layout
        {
            const int e = tid & (TM - 1), half = tid >> 7;              // THREADS == 2 * TM
            float x[OU];
#pragma unroll
            for (int o = 0; o < OU; o++) x[o] = (OT || o < O) ? xs[o * TM + e] : 0.f;
            const int nk4 = H1 >> 2, k_lo = half ? (nk4 + 1) / 2 : 0, k_hi = half ? nk4 : (nk4 + 1) / 2;
            uint8_t* dst = Asm + (e >> 3) * 128 + (e & 7) * 16;
#pragma unroll 2
            for (int k4 = k_lo; k4 < k_hi; k4++) {
                float4 s4 = *reinterpret_cast<const float4*>(b1 + 4 * k4);
#pragma unroll
                for (int o = 0; o < OU; o++) {
                    if (OT || o < O) {
                        const float4 w = *reinterpret_cast<const float4*>(W1 + o * H1 + 4 * k4);
                        s4.x = fmaf(x[o], w.x, s4.x); s4.y = fmaf(x[o], w.y, s4.y); s4.z = fmaf(x[o], w.z, s4.z); s4.w = fmaf(x[o], w.w, s4.w);
                    }
                }
                *reinterpret_cast<float4*>(dst + (size_t)k4 * LBO_A) =
                    make_float4(to_tf32(fmaxf(s4.x, 0.f)), to_tf32(fmaxf(s4.y, 0.f)), to_tf32(fmaxf(s4.z, 0.f)), to_tf32(fmaxf(s4.w, 0.f)));
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // A: generic-proxy writes -> tensor-core (async proxy) reads
        __syncthreads();
        float d[NCH][8];                                    // this warpgroup's accumulators, column chunk ch = columns 16 ch ..
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
        for (int kb = 0; kb < (H1 >> 3); kb++) {
            const uint64_t da = smem_desc(a_addr + (uint32_t)kb * 2u * LBO_A, LBO_A, 128u);
#pragma unroll
            for (int ch = 0; ch < NCH; ch++)
                if (ch < nch) wgmma_tf32_n16(d[ch], da, smem_desc(b_addr + (uint32_t)ch * 256u + (uint32_t)kb * 2u * LBO_B, LBO_B, 128u), kb > 0 ? 1u : 0u);
        }
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        if (tile + (int)gridDim.x < ntiles) load_obs(tile + gridDim.x);      // xs is free again: next tile's loads fly during the MMAs
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        auto epilogue = [&](auto ao_tag) {
            constexpr int AC = decltype(ao_tag)::value;          // head width at compile time (0: generic, predicated up to AG_MAX_A)
            constexpr int AU = AC ? AC : AG_MAX_A;
            // accumulator layout of m64nNk8: warp w of the warpgroup holds rows 16 (w % 4) + lane / 4 and + 8; within each group of
            // 8 columns, lane % 4 holds columns 2 (lane % 4) and + 1.  s[0] / s[1]: head partial sums of the two rows.
            float s[2][AU];
#pragma unroll
            for (int a = 0; a < AU; a++) { s[0][a] = 0.f; s[1][a] = 0.f; }
#pragma unroll
            for (int ch = 0; ch < NCH; ch++) {
                if (ch >= nch) break;
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    const int n = 16 * ch + 8 * j + 2 * (lane & 3);
                    if (n < H2) {                                       // H2 is a multiple of 4: n + 1 < H2 as well
                        const float2 bb = *reinterpret_cast<const float2*>(b2 + n);
                        const float* w3a = W3 + n * AO;
                        const float* w3b = w3a + AO;
#pragma unroll
                        for (int r = 0; r < 2; r++) {
                            const float h0 = fmaxf(d[ch][4 * j + 2 * r] + bb.x, 0.f), h1v = fmaxf(d[ch][4 * j + 2 * r + 1] + bb.y, 0.f);
#pragma unroll
                            for (int a = 0; a < AU; a++)
                                if (AC || a < AO) s[r][a] = fmaf(h1v, w3b[a], fmaf(h0, w3a[a], s[r][a]));
                        }
                    }
                }
            }
#pragma unroll
            for (int r = 0; r < 2; r++)
#pragma unroll
                for (int a = 0; a < AU; a++) {
                    s[r][a] += __shfl_xor_sync(0xffffffffu, s[r][a], 1);
                    s[r][a] += __shfl_xor_sync(0xffffffffu, s[r][a], 2);
                }
            const int r = lane & 3;                                     // lanes 0 / 1 of each quad finish row 0 / 1
            const int env = e0 + 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * r;
            if (r < 2 && env < P.n) {
                float sh[AU];
#pragma unroll
                for (int a = 0; a < AU; a++) sh[a] = (AC || a < AO) ? b3[a] + (r ? s[1][a] : s[0][a]) : 0.f;
                head_outputs<AC>(P, net, A, env, step, sh, b3 + AO);
            }
        };
        if (net == 1) epilogue(std::integral_constant<int, 1>{});
        else epilogue(std::integral_constant<int, AT>{});
    }
}

// StreamingNormalize.update for the observation columns and the reward column in one launch (normalize.py:73-99):
// per column j: S1 = sum(x - mean), S2 = sum((x - mean)^2) over the batch (block partials, then the last block to
// finish adds them in a fixed order -> bit-reproducible); count += n; new_mean = mean + S1/count;
// var_sum += S2 - S1^2/count  ( = sum (x - mean)(x - new_mean) ).
struct ExperienceArgs { AgentDev D; const float* __restrict__ observ; const float* __restrict__ reward; int n; float* sums_out; };

// finalisation shared by the single-GPU kernel and the sharded path (sums = [O+1][2] (S1, S2) over ALL ranks, n_total likewise)
__device__ __forceinline__ void filters_finalize(const AgentDev& D, int col, float s1, float s2, int n_total, float first_value) {
    const int O = D.cfg.obs_dim;
    const int which = col < O ? 0 : 1;
    const int64_t cnt = D.cnt[which] + n_total;
    const float step = (float)cnt;
    float* meanp = filt_mean(D.filt, O, col);
    float* varp = filt_var_sum(D.filt, O, col);
    float new_mean = *meanp + s1 / step;
    if (cnt <= 1) new_mean = first_value;                                   // tf.cond(count > 1, new_mean, value[0])
    *varp += s2 - s1 * (s1 / step);
    *meanp = new_mean;
}

__global__ void __launch_bounds__(256) experience_kernel(const ExperienceArgs P) {
    const int O = P.D.cfg.obs_dim, C = O + 1;
    __shared__ float red[2 * (AG_MAX_O + 1)][8];
    __shared__ float mean_s[AG_MAX_O + 1];
    __shared__ int last;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < C) mean_s[tid] = *filt_mean(P.D.filt, O, tid);
    __syncthreads();
    // each thread walks rows with a fixed stride; column sums kept per thread for its own column set
    for (int cidx = 0; cidx < C; cidx++) {
        float s1 = 0.f, s2 = 0.f;
        const float m = mean_s[cidx];
        for (int e = blockIdx.x * blockDim.x + tid; e < P.n; e += gridDim.x * blockDim.x) {
            const float x = cidx < O ? P.observ[(size_t)e * O + cidx] : P.reward[e];
            const float d = x - m;
            s1 += d; s2 = fmaf(d, d, s2);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
        if (lane == 0) { red[2 * cidx][warp] = s1; red[2 * cidx + 1][warp] = s2; }
    }
    __syncthreads();
    if (tid < 2 * C) {
        float s = 0.f;
        for (int w = 0; w < 8; w++) s += red[tid][w];
        P.D.partial[(size_t)blockIdx.x * 2 * C + tid] = s;
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) last = (atomicAdd(reinterpret_cast<unsigned long long*>(&P.D.cnt[3]), 1ull) == (unsigned long long)gridDim.x - 1);
    __syncthreads();
    if (!last) return;
    __threadfence();
    if (tid < C) {
        float s1 = 0.f, s2 = 0.f;
        for (int b = 0; b < (int)gridDim.x; b++) {
            s1 += __ldcg(&P.D.partial[(size_t)b * 2 * C + 2 * tid]);
            s2 += __ldcg(&P.D.partial[(size_t)b * 2 * C + 2 * tid + 1]);
        }
        if (P.sums_out) { P.sums_out[2 * tid] = s1; P.sums_out[2 * tid + 1] = s2; }          // sharded: another rank's sums are added first
        else filters_finalize(P.D, tid, s1, s2, P.n, tid < O ? P.observ[tid] : P.reward[0]);
    }
    __syncthreads();
    if (tid == 0) {
        if (!P.sums_out) advance_counts(P.D, P.n);
        P.D.cnt[3] = 0;
    }
}

// sharded rollouts: sums = this rank's partial sums after an all-reduce(sum) over the ranks; n_total = envs of all ranks
__global__ void experience_finalize_kernel(const AgentDev D, const float* __restrict__ sums, int n_total,
                                           const float* __restrict__ observ, const float* __restrict__ reward) {
    const int O = D.cfg.obs_dim, tid = threadIdx.x;
    if (tid <= O) filters_finalize(D, tid, sums[2 * tid], sums[2 * tid + 1], n_total, tid < O ? observ[tid] : reward[0]);
    __syncthreads();
    if (tid == 0) advance_counts(D, n_total);
}

__global__ void transform_reward_kernel(const AgentDev D, const float* __restrict__ r, int n, float* __restrict__ out) {
    const float inv = filter_inv_std(*filt_var_sum(D.filt, D.cfg.obs_dim, D.cfg.obs_dim), D.cnt[1]);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        out[i] = fminf(fmaxf(r[i] * inv, -D.cfg.reward_clip), D.cfg.reward_clip);      // center=False, scale=True, clip=10
}

// ---- scans ---------------------------------------------------------------------------------------------------------
// one thread per episode row, walking backwards in time; rows are laid out by (stride_e, stride_t) so a time-major
// buffer (stride_e = 1) is read fully coalesced
// The recurrences are serial in time but every load is independent of them: each thread fetches SCAN_U time steps into
// registers first (SCAN_U x 2-3 loads in flight per thread), then runs the dependent chain -- without this the kernel waits
// one DRAM latency per time step.
constexpr int SCAN_U = 8;

template <bool ADV>
__global__ void __launch_bounds__(256) row_scan_kernel(const float* __restrict__ reward, const float* __restrict__ value,
                                                       const int32_t* __restrict__ length, int episodes, int L,
                                                       int64_t se, int64_t st, float discount, float* __restrict__ out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= episodes) return;
    const int len = length[e];
    float agg = 0.f, next_v = 0.f;                           // value[:, 1:] padded with zeros (utility.py:116)
    const int64_t base = (int64_t)e * se;
    for (int t1 = L; t1 > 0; t1 -= SCAN_U) {
        float r[SCAN_U], v[SCAN_U];
#pragma unroll
        for (int u = 0; u < SCAN_U; u++) {
            const int t = t1 - 1 - u;
            r[u] = t >= 0 ? reward[base + (int64_t)t * st] : 0.f;
            v[u] = (ADV && t >= 0) ? value[base + (int64_t)t * st] : 0.f;
        }
#pragma unroll
        for (int u = 0; u < SCAN_U; u++) {
            const int t = t1 - 1 - u;
            if (t < 0) break;
            float cur;
            if (ADV) { cur = (t < len) ? r[u] + discount * next_v - v[u] : 0.f; next_v = v[u]; }   // mask * delta
            else cur = (t < len) ? r[u] : 0.f;                                                     // mask * reward
            agg = cur + discount * agg;
            out[base + (int64_t)t * st] = agg;
        }
    }
}

__global__ void __launch_bounds__(256) gae_segments_kernel(const float* __restrict__ reward, const float* __restrict__ value,
                                                           const uint8_t* __restrict__ done, int T, int n, float discount,
                                                           float lambda, float* __restrict__ out_ret, float* __restrict__ out_adv) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    float next_v = value[(size_t)T * n + e], ret = next_v, adv = 0.f;
    for (int t1 = T; t1 > 0; t1 -= SCAN_U) {
        float r[SCAN_U], v[SCAN_U]; uint8_t d[SCAN_U];
#pragma unroll
        for (int u = 0; u < SCAN_U; u++) {
            const int t = t1 - 1 - u;
            const size_t idx = (size_t)(t >= 0 ? t : 0) * n + e;
            r[u] = reward[idx]; v[u] = value[idx]; d[u] = done[idx];
        }
#pragma unroll
        for (int u = 0; u < SCAN_U; u++) {
            const int t = t1 - 1 - u;
            if (t < 0) break;
            const size_t idx = (size_t)t * n + e;
            const float nd = d[u] ? 0.f : 1.f;
            const float delta = r[u] + discount * next_v * nd - v[u];
            adv = delta + discount * lambda * nd * adv;
            ret = r[u] + discount * nd * ret;
            if (out_adv) out_adv[idx] = adv;
            if (out_ret) out_ret[idx] = ret;
            next_v = v[u];
        }
    }
}

}  // namespace rexsim

using namespace rexsim;

struct RexAgent {
    AgentDev D;                        // filt, cnt and partial are allocated from `mem` in place
    DeviceBuffers mem;
    float* params = nullptr;           // what D.params reads (the kernels' pointer is to const)
    int sm_count = 132;
    int64_t launches = 0;
    int precision = 0;                 // 0: fp32 on the CUDA cores (parity default); 1: layer 2 on the tensor cores in TF32
};

struct RexRnn {
    RexAgent* agent;                   // filters, step counter and value network
    RexRnnConfig cfg;
    DeviceBuffers mem;
    float* params = nullptr;           // the policy block
    float* state = nullptr;            // GRU: [num_envs][cell]
    int64_t floats = 0;
    int64_t launches = 0;
};

// the instance compiled for this network's input / output widths (the reference's tasks: 4 or 16 observations, 1-8 actions)
typedef void (*PerformTcKernel)(const PerformArgs);
static PerformTcKernel perform_tc_pick(const RexAgentConfig* c) {
    const int O = c->obs_dim, A = c->action_dim;
    if (O == 4) { if (A == 1) return perform_tc_kernel<4, 1>; if (A == 2) return perform_tc_kernel<4, 2>; if (A == 8) return perform_tc_kernel<4, 8>; return perform_tc_kernel<4, 0>; }
    if (O == 16) { if (A == 2) return perform_tc_kernel<16, 2>; if (A == 4) return perform_tc_kernel<16, 4>; return perform_tc_kernel<16, 0>; }
    return perform_tc_kernel<0, 0>;
}

static int check_cfg(const RexAgentConfig* c) {
    if (!c) return fail(REXSIM_ERR_INVALID, "null agent config");
    if (c->obs_dim <= 0 || c->obs_dim > AG_MAX_O || c->action_dim <= 0 || c->action_dim > AG_MAX_A)
        return fail(REXSIM_ERR_INVALID, "agent: obs_dim must be 1..32 and action_dim 1..8");
    if (c->hidden1 <= 0 || c->hidden1 > AG_MAX_H1 || c->hidden2 <= 0 || c->hidden2 > AG_MAX_H2 || (c->hidden1 & 3) || (c->hidden2 & 3))
        return fail(REXSIM_ERR_UNSUPPORTED, "agent: hidden1 <= 256, hidden2 <= 128, both multiples of 4");
    return REXSIM_OK;
}

// StreamingNormalize.update of one batch; sums_out null: into the filters, else this rank's partial sums for the sharded path
static int experience(RexAgent* a, const float* observ, const float* reward, int32_t n, float* sums_out, void* stream) {
    if (n <= 0) return fail(REXSIM_ERR_INVALID, "agent: n must be positive");
    ExperienceArgs P; P.D = a->D; P.observ = observ; P.reward = reward; P.n = n; P.sums_out = sums_out;
    int blocks = (n + 255) / 256;
    if (blocks > RED_BLOCKS) blocks = RED_BLOCKS;
    experience_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(P);
    return enqueue(a, cudaGetLastError(), "experience launch");
}

// discounted_return (ADV = false, no values) / lambda_advantage; the scans have no handle, so they count no launch
template <bool ADV>
static int row_scan(const float* reward, const float* value, const int32_t* length, int32_t episodes, int32_t L, int64_t se,
                    int64_t st, float discount, float* out, void* stream) {
    if (!reward || (ADV && !value) || !length || !out) return fail(REXSIM_ERR_INVALID, "null argument");
    if (episodes <= 0 || L <= 0) return fail(REXSIM_ERR_INVALID, "agent: empty scan");
    row_scan_kernel<ADV><<<(episodes + 255) / 256, 256, 0, (cudaStream_t)stream>>>(reward, value, length, episodes, L, se, st, discount, out);
    CK(cudaGetLastError());
    return REXSIM_OK;
}

extern "C" {

int64_t rexagent_policy_floats(const RexAgentConfig* c) {
    return c ? param_layout(c->obs_dim, c->action_dim, c->hidden1, c->hidden2, true).floats : 0;
}
int64_t rexagent_value_floats(const RexAgentConfig* c) {
    return c ? param_layout(c->obs_dim, c->action_dim, c->hidden1, c->hidden2, false).floats : 0;
}

static size_t perform_smem_bytes(const RexAgentConfig* c, int tm) {
    const int64_t p = rexagent_policy_floats(c), v = rexagent_value_floats(c);
    return perform_smem((int)(p > v ? p : v), c->hidden1, tm).bytes;
}

int rexagent_create(const RexAgentConfig* cfg, RexAgent** out) {
    int rc = check_cfg(cfg);
    if (rc) return rc;
    if (!out) return fail(REXSIM_ERR_INVALID, "null argument");
    if (perform_smem_bytes(cfg, 128) > 227 * 1024) return fail(REXSIM_ERR_UNSUPPORTED, "agent: network does not fit the 227 KB of shared memory");
    if (cfg->action_dim * (cfg->hidden2 / 4) > cfg->hidden1) return fail(REXSIM_ERR_UNSUPPORTED, "agent: action_dim * hidden2 / 4 must not exceed hidden1");
    RexAgent* a = new RexAgent();
    struct Guard { RexAgent* a; ~Guard() { if (a) rexagent_destroy(a); } } guard{a};  // frees everything on an early return
    a->D.cfg = *cfg;
    a->D.pol_floats = (int)rexagent_policy_floats(cfg); a->D.val_floats = (int)rexagent_value_floats(cfg);
    const size_t np = (size_t)a->D.pol_floats + a->D.val_floats;
    const int O = cfg->obs_dim;
    int dev = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&a->sm_count, cudaDevAttrMultiProcessorCount, dev));
    if (a->mem.zeroed(&a->params, np) || a->mem.zeroed(&a->D.filt, 2 * O + 2) || a->mem.zeroed(&a->D.cnt, 4) ||
        a->mem.zeroed(&a->D.partial, (size_t)RED_BLOCKS * 2 * (O + 1)))
        return REXSIM_ERR_CUDA;
    a->D.params = a->params;
    CK(cudaFuncSetAttribute(perform_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)perform_smem_bytes(cfg, 64)));
    CK(cudaFuncSetAttribute(perform_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)perform_smem_bytes(cfg, 128)));
    CK(cudaDeviceSynchronize());
    guard.a = nullptr;
    *out = a;
    return REXSIM_OK;
}
void rexagent_destroy(RexAgent* a) {
    if (!a) return;
    a->mem.release();
    delete a;
}
int rexagent_set_precision(RexAgent* a, int32_t mode) {
    if (!a) return fail(REXSIM_ERR_INVALID, "null argument");
    if (mode != 0 && mode != 1) return fail(REXSIM_ERR_INVALID, "agent: precision must be 0 (fp32) or 1 (tf32 tensor cores)");
    if (mode == 1) {
        const RexAgentConfig* c = &a->D.cfg;
        if ((c->hidden1 & 7) || c->obs_dim > 16 || perform_tc_smem_bytes(c) > 227 * 1024)
            return fail(REXSIM_ERR_UNSUPPORTED, "agent: the tensor-core path needs hidden1 % 8 == 0, obs_dim <= 16 and operands that fit 227 KB of shared memory");
        CK(cudaFuncSetAttribute(perform_tc_pick(c), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)perform_tc_smem_bytes(c)));
    }
    a->precision = mode;
    return REXSIM_OK;
}
int rexagent_set_params(RexAgent* a, const float* h, int64_t n) {
    if (!a || !h) return fail(REXSIM_ERR_INVALID, "null argument");
    if (n != (int64_t)a->D.pol_floats + a->D.val_floats) return fail(REXSIM_ERR_INVALID, "agent: parameter block size mismatch");
    CK(cudaMemcpy(a->params, h, n * sizeof(float), cudaMemcpyHostToDevice));
    return REXSIM_OK;
}
int rexagent_get_params(RexAgent* a, float* h, int64_t n) {
    if (!a || !h) return fail(REXSIM_ERR_INVALID, "null argument");
    if (n != (int64_t)a->D.pol_floats + a->D.val_floats) return fail(REXSIM_ERR_INVALID, "agent: parameter block size mismatch");
    CK(cudaMemcpy(h, a->params, n * sizeof(float), cudaMemcpyDeviceToHost));
    return REXSIM_OK;
}
int rexagent_params_buffer(RexAgent* a, float** p) {
    if (!a || !p) return fail(REXSIM_ERR_INVALID, "null argument");
    *p = a->params;
    return REXSIM_OK;
}
int rexagent_state_buffers(RexAgent* a, float** filt, int64_t** counters) {
    if (!a) return fail(REXSIM_ERR_INVALID, "null argument");
    if (filt) *filt = a->D.filt;
    if (counters) *counters = a->D.cnt;
    return REXSIM_OK;
}
int rexagent_set_filters(RexAgent* a, int64_t oc, const float* om, const float* ov, int64_t rc, float rm, float rv) {
    if (!a || !om || !ov) return fail(REXSIM_ERR_INVALID, "null argument");
    const int O = a->D.cfg.obs_dim;
    std::vector<float> f(2 * O + 2);
    for (int i = 0; i < O; i++) { f[i] = om[i]; f[O + i] = ov[i]; }
    f[2 * O] = rm; f[2 * O + 1] = rv;
    int64_t c[4] = {oc, rc, 0, 0};
    CK(cudaMemcpy(a->D.filt, f.data(), f.size() * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(a->D.cnt, c, sizeof(c), cudaMemcpyHostToDevice));
    return REXSIM_OK;
}
int rexagent_get_filters(RexAgent* a, int64_t* counts, float* om, float* ov, float* rmv) {
    if (!a || !counts || !om || !ov || !rmv) return fail(REXSIM_ERR_INVALID, "null argument");
    const int O = a->D.cfg.obs_dim;
    std::vector<float> f(2 * O + 2);
    int64_t c[4];
    CK(cudaMemcpy(f.data(), a->D.filt, f.size() * sizeof(float), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(c, a->D.cnt, sizeof(c), cudaMemcpyDeviceToHost));
    for (int i = 0; i < O; i++) { om[i] = f[i]; ov[i] = f[O + i]; }
    rmv[0] = f[2 * O]; rmv[1] = f[2 * O + 1];
    counts[0] = c[0]; counts[1] = c[1];
    return REXSIM_OK;
}

// the arguments of one perform call (net_base 0: perform_kernel's blockIdx.y picks the network)
static PerformArgs perform_args(const RexAgent* a, const float* observ, int32_t n, int32_t training, uint64_t seed, uint32_t step,
                                uint32_t env_offset, float* action, float* mean, float* logprob, float* value, float* observ_copy) {
    PerformArgs P;
    P.D = a->D; P.observ = observ; P.n = n; P.training = training; P.net_base = 0; P.seed = seed; P.step = step;
    P.env_offset = env_offset; P.action = action; P.mean = mean; P.logprob = logprob; P.value = value; P.observ_copy = observ_copy;
    return P;
}

// perform_kernel on `nets` networks from P.net_base, at most `ctas` persistent CTAs per network: 64-env tiles while there are
// fewer 128-env tiles than CTAs, so that more SMs get a tile, 128-env tiles (8 x 4 register tile per thread) above
static void perform_fp32_launch(const RexAgent* a, const PerformArgs& P, int ctas, int nets, cudaStream_t st) {
    const int tm = (P.n + 127) / 128 >= ctas ? 128 : 64;
    const int ntiles = (P.n + tm - 1) / tm;
    const dim3 grid(ntiles < ctas ? ntiles : ctas, nets);
    const int threads = 16 * (a->D.cfg.hidden2 / 4) > tm ? 16 * (a->D.cfg.hidden2 / 4) : tm;
    if (tm == 128) perform_kernel<128><<<grid, threads, perform_smem_bytes(&a->D.cfg, 128), st>>>(P);
    else perform_kernel<64><<<grid, threads, perform_smem_bytes(&a->D.cfg, 64), st>>>(P);
}

int rexagent_perform(RexAgent* a, const float* observ, int32_t n, int32_t training, uint64_t seed, uint32_t step,
                     uint32_t env_offset, float* action, float* mean, float* logprob, float* value, float* observ_copy,
                     void* stream) {
    if (!a || !observ) return fail(REXSIM_ERR_INVALID, "null argument");
    if (n <= 0) return fail(REXSIM_ERR_INVALID, "agent: n must be positive");
    const PerformArgs P = perform_args(a, observ, n, training, seed, step, env_offset, action, mean, logprob, value, observ_copy);
    // one CTA per SM (the weights fill most of the shared memory); the two networks run in different CTAs (blockIdx.y), on
    // half the SMs each.  The wgmma path always uses 128-env tiles.
    const int half = a->sm_count / 2 > 0 ? a->sm_count / 2 : 1;
    const cudaStream_t st = (cudaStream_t)stream;
    if (a->precision == 1) {
        const int ntiles = (n + 127) / 128;
        perform_tc_pick(&a->D.cfg)<<<dim3(ntiles < half ? ntiles : half, 2), tc::THREADS, perform_tc_smem_bytes(&a->D.cfg), st>>>(P);
    } else {
        perform_fp32_launch(a, P, half, 2, st);
    }
    return enqueue(a, cudaGetLastError(), "perform launch");
}
int rexagent_experience(RexAgent* a, const float* observ, const float* reward, int32_t n, void* stream) {
    if (!a || !observ || !reward) return fail(REXSIM_ERR_INVALID, "null argument");
    return experience(a, observ, reward, n, nullptr, stream);
}
int rexagent_experience_partial(RexAgent* a, const float* observ, const float* reward, int32_t n, float* sums, void* stream) {
    if (!a || !observ || !reward || !sums) return fail(REXSIM_ERR_INVALID, "null argument");
    return experience(a, observ, reward, n, sums, stream);
}
int rexagent_experience_finalize(RexAgent* a, const float* sums, int32_t n_total, const float* observ, const float* reward, void* stream) {
    if (!a || !sums || !observ || !reward) return fail(REXSIM_ERR_INVALID, "null argument");
    if (n_total <= 0) return fail(REXSIM_ERR_INVALID, "agent: n_total must be positive");
    experience_finalize_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(a->D, sums, n_total, observ, reward);
    return enqueue(a, cudaGetLastError(), "experience_finalize launch");
}
int rexagent_transform_reward(RexAgent* a, const float* reward, int32_t n, float* out, void* stream) {
    if (!a || !reward || !out) return fail(REXSIM_ERR_INVALID, "null argument");
    if (n <= 0) return REXSIM_OK;
    int blocks = (n + 255) / 256;
    if (blocks > 1184) blocks = 1184;
    transform_reward_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(a->D, reward, n, out);
    return enqueue(a, cudaGetLastError(), "transform_reward launch");
}
int rexagent_discounted_return(const float* reward, const int32_t* length, int32_t episodes, int32_t L, int64_t se, int64_t st,
                               float discount, float* out, void* stream) {
    return row_scan<false>(reward, nullptr, length, episodes, L, se, st, discount, out, stream);
}
int rexagent_lambda_advantage(const float* reward, const float* value, const int32_t* length, int32_t episodes, int32_t L,
                              int64_t se, int64_t st, float discount, float* out, void* stream) {
    return row_scan<true>(reward, value, length, episodes, L, se, st, discount, out, stream);
}
int rexagent_gae_segments(const float* reward, const float* value, const uint8_t* done, int32_t T, int32_t n, float discount,
                          float lambda, float* out_return, float* out_advantage, void* stream) {
    if (!reward || !value || !done) return fail(REXSIM_ERR_INVALID, "null argument");
    if (T <= 0 || n <= 0) return fail(REXSIM_ERR_INVALID, "agent: empty scan");
    gae_segments_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(reward, value, done, T, n, discount, lambda, out_return, out_advantage);
    CK(cudaGetLastError());
    return REXSIM_OK;
}
int64_t rexagent_launch_count(const RexAgent* a) { return a ? a->launches : 0; }

// ---- include/rexsim_recurrent.h ------------------------------------------------------------------------------------------
int64_t rexrnn_policy_floats(const RexAgentConfig* c, const RexRnnConfig* r) {
    if (!c || !r) return 0;
    if (r->kind == REXRNN_LINEAR) return linear_floats(c->obs_dim, c->action_dim);
    return rnn_layout<int64_t>(c->obs_dim, c->action_dim, r->hidden1, r->cell).floats;
}
int rexrnn_check(const RexAgentConfig* c, const RexRnnConfig* r) {
    int rc = check_cfg(c);
    if (rc) return rc;
    if (!r) return fail(REXSIM_ERR_INVALID, "null recurrent config");
    if (r->kind != REXRNN_GRU && r->kind != REXRNN_LINEAR) return fail(REXSIM_ERR_INVALID, "rnn: kind must be REXRNN_GRU or REXRNN_LINEAR");
    if (r->num_envs <= 0) return fail(REXSIM_ERR_INVALID, "rnn: num_envs must be positive");
    if (r->kind == REXRNN_GRU) {
        if (r->hidden1 <= 0 || r->hidden1 > RNN_MAX_H1 || r->cell <= 0 || r->cell > RNN_MAX_G || (r->hidden1 & 3) || (r->cell & 3))
            return fail(REXSIM_ERR_UNSUPPORTED, "rnn: hidden1 <= 256, cell <= 128, both multiples of 4");
        if (rnn_smem(c->obs_dim, r->hidden1, r->cell).bytes > 227 * 1024)       // 174 KB at the largest accepted shape
            return fail(REXSIM_ERR_UNSUPPORTED, "rnn: the cell's tile does not fit the 227 KB of shared memory");
    }
    return REXSIM_OK;
}
int rexrnn_create(RexAgent* a, const RexRnnConfig* cfg, RexRnn** out) {
    if (!a || !out) return fail(REXSIM_ERR_INVALID, "null argument");
    int rc = rexrnn_check(&a->D.cfg, cfg);
    if (rc) return rc;
    RexRnn* r = new RexRnn();
    struct Guard { RexRnn* r; ~Guard() { if (r) rexrnn_destroy(r); } } guard{r};
    r->agent = a; r->cfg = *cfg;
    r->floats = rexrnn_policy_floats(&a->D.cfg, cfg);
    if (r->mem.zeroed(&r->params, (size_t)r->floats)) return REXSIM_ERR_CUDA;
    if (cfg->kind == REXRNN_GRU) {
        if (r->mem.zeroed(&r->state, (size_t)cfg->num_envs * cfg->cell)) return REXSIM_ERR_CUDA;
        CK(cudaFuncSetAttribute(gru_policy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)rnn_smem(a->D.cfg.obs_dim, cfg->hidden1, cfg->cell).bytes));
    }
    CK(cudaDeviceSynchronize());
    guard.r = nullptr;
    *out = r;
    return REXSIM_OK;
}
void rexrnn_destroy(RexRnn* r) {
    if (!r) return;
    r->mem.release();
    delete r;
}
int rexrnn_set_params(RexRnn* r, const float* h, int64_t n) {
    if (!r || !h) return fail(REXSIM_ERR_INVALID, "null argument");
    if (n != r->floats) return fail(REXSIM_ERR_INVALID, "rnn: parameter block size mismatch");
    CK(cudaMemcpy(r->params, h, n * sizeof(float), cudaMemcpyHostToDevice));
    return REXSIM_OK;
}
int rexrnn_get_params(RexRnn* r, float* h, int64_t n) {
    if (!r || !h) return fail(REXSIM_ERR_INVALID, "null argument");
    if (n != r->floats) return fail(REXSIM_ERR_INVALID, "rnn: parameter block size mismatch");
    CK(cudaMemcpy(h, r->params, n * sizeof(float), cudaMemcpyDeviceToHost));
    return REXSIM_OK;
}
int rexrnn_state_buffer(RexRnn* r, float** state) {
    if (!r || !state) return fail(REXSIM_ERR_INVALID, "null argument");
    *state = r->state;
    return REXSIM_OK;
}
int rexrnn_perform(RexRnn* r, const float* observ, const uint8_t* begin, int32_t n, int32_t training, uint64_t seed, uint32_t step,
                   uint32_t env_offset, float* action, float* mean, float* logprob, float* value, float* observ_copy, void* stream) {
    if (!r || !observ) return fail(REXSIM_ERR_INVALID, "null argument");
    if (n <= 0 || n > r->cfg.num_envs) return fail(REXSIM_ERR_INVALID, "rnn: n must be 1..num_envs");
    const bool policy = action || mean || logprob;
    if (observ_copy && !policy) return fail(REXSIM_ERR_INVALID, "rnn: observ_copy is written by the policy pass only");
    const RexAgent* a = r->agent;
    const cudaStream_t st = (cudaStream_t)stream;
    int launches = 0;
    if (policy) {
        RnnArgs R;
        R.P = perform_args(a, observ, n, training, seed, step, env_offset, action, mean, logprob, nullptr, observ_copy);
        R.params = r->params; R.state = r->state; R.begin = begin; R.H1 = r->cfg.hidden1; R.G = r->cfg.cell;
        if (r->cfg.kind == REXRNN_GRU) {
            const int ntiles = (n + RNN_TM - 1) / RNN_TM, threads = 4 * R.G > 128 ? 4 * R.G : 128;
            gru_policy_kernel<<<ntiles < a->sm_count ? ntiles : a->sm_count, threads,
                                rnn_smem(a->D.cfg.obs_dim, R.H1, R.G).bytes, st>>>(R);
        } else {
            linear_policy_kernel<<<(n + LIN_TM - 1) / LIN_TM, LIN_TM, 0, st>>>(R);
        }
        launches++;
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return cuda_fail(e, "rnn policy launch");
    }
    if (value) {                       // the agent's value network alone, on every SM
        PerformArgs P = perform_args(a, observ, n, training, seed, step, env_offset, nullptr, nullptr, nullptr, value, nullptr);
        P.net_base = 1;
        perform_fp32_launch(a, P, a->sm_count, 1, st);
        launches++;
    }
    return enqueue(r, cudaGetLastError(), "rnn value launch", launches);
}
int64_t rexrnn_launch_count(const RexRnn* r) { return r ? r->launches : 0; }

}  // extern "C"
