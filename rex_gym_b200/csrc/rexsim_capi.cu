// rexsim_capi.cu -- the C ABI declared in include/rexsim.h (plain pointers and sizes, no torch types).
#include "rexsim_kernel.cuh"
#include <cstdio>
#include <cstring>
#include <cmath>
#include <vector>

namespace rexsim {
cudaError_t launch_step(const Params& P, cudaStream_t st);
cudaError_t launch_reset(const Params& P, float* obs_out, cudaStream_t st);
cudaError_t launch_settle(const Params& P, float* snap_f, int32_t* snap_i, cudaStream_t st);
cudaError_t launch_get_state(const Params& P, float* out_f, int32_t* out_i, cudaStream_t st);
cudaError_t launch_set_state(const Params& P, const float* in_f, cudaStream_t st);
cudaError_t launch_rebalance(const int32_t* cost, int n, int32_t* hist, int32_t* perm, cudaStream_t st);
}  // namespace rexsim

using namespace rexsim;

struct RexSim {
    Params P;
    float* d_model = nullptr;
    float* d_sf = nullptr;
    int32_t* d_si = nullptr;
    float* d_snap_f = nullptr;
    int32_t* d_snap_i = nullptr;
    float* d_zoff = nullptr;
    int32_t* d_err = nullptr;
    float* d_cmd = nullptr;
    int32_t* d_perm = nullptr;         // slot -> env, sorted by solver cost (rexsim_rebalance)
    int32_t* d_cost = nullptr;
    int32_t* d_hist = nullptr;
    bool perm_valid = false;
    float* d_ring = nullptr;           // sensor history [D][words][N] (sensor model only)
    float* d_snap_ring = nullptr;      // [nsnap][D][words]
    float* d_act = nullptr;            // staging for rexsim_step_host
    uint8_t* d_out = nullptr;          // obs | reward | done (same layout as the host block)
    int A = 0, O = 0;
    int nsnap = 1;
    int64_t launches = 0;
    int32_t launched[3] = {0, 0, 0};   // step_kernel instance of the last step launch: BLOCK, OCC, SENSOR
};

static thread_local char g_err[512] = "";
namespace rexsim { void set_error(const char* msg) { snprintf(g_err, sizeof(g_err), "%s", msg); } }   // shared with rexsim_agent.cu
static int fail(int code, const char* msg) { snprintf(g_err, sizeof(g_err), "%s", msg); return code; }
static int cuda_fail(cudaError_t e, const char* where) {
    snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
    return REXSIM_ERR_CUDA;
}
#define CK(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return cuda_fail(_e, #x); } while (0)

extern "C" {

const char* rexsim_last_error(void) { return g_err; }

int rexsim_obs_dim(int32_t task, int32_t num_motors) { return obs_dim(task, num_motors); }
int rexsim_action_dim(int32_t task, int32_t signal) { return task_shape(task).act[signal == REXSIM_SIGNAL_IK ? 0 : 1]; }
int rexsim_state_words(const RexSimConfig* cfg, int32_t* n_float, int32_t* n_int) {
    if (!cfg) return fail(REXSIM_ERR_INVALID, "null config");
    if (n_float) *n_float = NF;
    if (n_int) *n_int = NI;
    return REXSIM_OK;
}

static int validate(const RexSimConfig* c) {
    if (c->num_envs <= 0) return fail(REXSIM_ERR_INVALID, "num_envs must be positive");
    if (c->task < 0 || c->task > 4 || c->signal < 0 || c->signal > 1) return fail(REXSIM_ERR_INVALID, "bad task/signal");
    if (c->num_motors != 12 && c->num_motors != 18) return fail(REXSIM_ERR_INVALID, "num_motors must be 12 (base) or 18 (arm)");
    if (c->num_motors == 18 && !(c->task == REXSIM_TASK_STANDUP || (c->task == REXSIM_TASK_WALK && c->signal == REXSIM_SIGNAL_IK)))
        return fail(REXSIM_ERR_UNSUPPORTED, "mark='arm' is built for the standup and walk-ik tasks");
    if (c->action_repeat <= 0 || c->solver_iterations <= 0 || !(c->sim_dt_d > 0)) return fail(REXSIM_ERR_INVALID, "bad time stepping");
    if (c->terrain == REXSIM_TERRAIN_RANDOM && (c->nfields <= 0 || !c->fields)) return fail(REXSIM_ERR_INVALID, "random terrain needs a heightfield bank");
    if (c->terrain != REXSIM_TERRAIN_PLANE && c->terrain != REXSIM_TERRAIN_RANDOM) return fail(REXSIM_ERR_UNSUPPORTED, "terrain type");
    if (c->toe_npts <= 0 || c->toe_npts > REXSIM_MAX_TOE_PTS) return fail(REXSIM_ERR_MODEL, "toe_npts out of range");
    if (!(c->gait_clock_scale > 0)) return fail(REXSIM_ERR_INVALID, "gait_clock_scale must be positive (1 = simulation clock)");
    if (!(c->control_latency >= 0) || !(c->pd_latency >= 0)) return fail(REXSIM_ERR_INVALID, "latencies must be >= 0");
    for (int k = 0; k < 5; k++) if (!(c->noise_stdev[k] >= 0)) return fail(REXSIM_ERR_INVALID, "noise_stdev must be >= 0");
    return REXSIM_OK;
}
static bool sensor_on(const RexSimConfig* c) {
    bool on = c->control_latency > 0 || c->pd_latency > 0;
    for (int k = 0; k < 5; k++) on = on || c->noise_stdev[k] > 0;
    return on;
}
int rexsim_history_depth(const RexSimConfig* c) {
    if (!c || !sensor_on(c)) return 0;
    // Rex._GetDelayedObservation reads history[n] and history[n + 1], n = int(latency / dt); once n + 1 reaches the deque's
    // length (maxlen 100, rex.py:122) it reads the oldest row instead
    const int n_ctl = (int)(c->control_latency / c->sim_dt_d), n_pd = (int)(c->pd_latency / c->sim_dt_d);
    const int n = n_ctl > n_pd ? n_ctl : n_pd;
    return n + 1 >= HIST_MAXLEN ? (int)HIST_MAXLEN : n + 2;
}
float rexsim_noise(uint64_t seed, uint32_t global_env, uint32_t reset_count, uint32_t control_step, uint32_t site, uint32_t comp) {
    return noise_unit(seed, global_env, reset_count, control_step, site, comp);
}

int rexsim_create(const RexSimConfig* cfg, const float* model_tables, int32_t n_model_floats, RexSim** out) {
    if (!cfg || !model_tables || !out) return fail(REXSIM_ERR_INVALID, "null argument");
    int rc = validate(cfg);
    if (rc) return rc;
    const int mt_floats = cfg->num_motors == 18 ? REXSIM_MT_FLOATS_ARM : REXSIM_MT_FLOATS;
    if (n_model_floats != mt_floats) return fail(REXSIM_ERR_MODEL, "model table size mismatch");
    RexSim* s = new RexSim();
    struct Guard { RexSim* s; ~Guard() { if (s) rexsim_destroy(s); } } guard{s};      // frees everything on an early return
    memset(&s->P, 0, sizeof(Params));
    s->P.cfg = *cfg;
    s->P.cfg.sim_dt = (float)cfg->sim_dt_d;
    const int N = cfg->num_envs;
    s->P.N = N;
    {
        int dev = 0, sms = 132;
        CK(cudaGetDevice(&dev));
        CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        s->P.sm_count = sms;
    }
    s->nsnap = cfg->terrain == REXSIM_TERRAIN_RANDOM ? cfg->nfields : 1;
    CK(cudaMalloc(&s->d_model, mt_floats * sizeof(float)));
    CK(cudaMemcpy(s->d_model, model_tables, mt_floats * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaMalloc(&s->d_sf, (size_t)NF * N * sizeof(float)));
    CK(cudaMalloc(&s->d_si, (size_t)NI * N * sizeof(int32_t)));
    CK(cudaMemset(s->d_sf, 0, (size_t)NF * N * sizeof(float)));
    CK(cudaMemset(s->d_si, 0, (size_t)NI * N * sizeof(int32_t)));
    CK(cudaMalloc(&s->d_snap_f, (size_t)NF * s->nsnap * sizeof(float)));
    CK(cudaMalloc(&s->d_snap_i, (size_t)NI * s->nsnap * sizeof(int32_t)));
    CK(cudaMemset(s->d_snap_f, 0, (size_t)NF * s->nsnap * sizeof(float)));
    CK(cudaMemset(s->d_snap_i, 0, (size_t)NI * s->nsnap * sizeof(int32_t)));
    CK(cudaMalloc(&s->d_err, (size_t)(N + 1) * sizeof(int32_t)));   /* [N] per-env bits + 1 word: OR of all */
    CK(cudaMemset(s->d_err, 0, (size_t)(N + 1) * sizeof(int32_t)));
    CK(cudaMalloc(&s->d_cmd, (size_t)cfg->num_motors * N * sizeof(float)));
    CK(cudaMemset(s->d_cmd, 0, (size_t)cfg->num_motors * N * sizeof(float)));
    CK(cudaMalloc(&s->d_perm, (size_t)N * sizeof(int32_t)));
    CK(cudaMalloc(&s->d_cost, (size_t)N * sizeof(int32_t)));
    CK(cudaMemset(s->d_cost, 0, (size_t)N * sizeof(int32_t)));
    CK(cudaMalloc(&s->d_hist, 256 * sizeof(int32_t)));
    if (sensor_on(cfg)) {
        Params& P = s->P;
        const double dt = cfg->sim_dt_d;
        P.sensor_on = 1;
        P.ring_depth = rexsim_history_depth(cfg);
        P.n_ctl = (int)(cfg->control_latency / dt); P.n_pd = (int)(cfg->pd_latency / dt);
        P.a_ctl = (float)((cfg->control_latency - P.n_ctl * dt) / dt); P.a_pd = (float)((cfg->pd_latency - P.n_pd * dt) / dt);
        P.lat_ctl = (float)cfg->control_latency; P.lat_pd = (float)cfg->pd_latency;
        for (int k = 0; k < 5; k++) P.noise_sd[k] = (float)cfg->noise_stdev[k];
        const size_t words = cfg->num_motors == 18 ? HW_WORDS_ARM : HW_WORDS;
        CK(cudaMalloc(&s->d_ring, (size_t)P.ring_depth * words * N * sizeof(float)));
        CK(cudaMemset(s->d_ring, 0, (size_t)P.ring_depth * words * N * sizeof(float)));
        CK(cudaMalloc(&s->d_snap_ring, (size_t)s->nsnap * P.ring_depth * words * sizeof(float)));
        CK(cudaMemset(s->d_snap_ring, 0, (size_t)s->nsnap * P.ring_depth * words * sizeof(float)));
        P.ring = s->d_ring; P.snap_ring = s->d_snap_ring;
    }
    s->A = rexsim_action_dim(cfg->task, cfg->signal); s->O = rexsim_obs_dim(cfg->task, cfg->num_motors);
    CK(cudaMalloc(&s->d_act, (size_t)N * s->A * sizeof(float)));
    CK(cudaMalloc(&s->d_out, (size_t)rexsim_host_out_bytes(s)));
    CK(cudaMemset(s->d_out, 0, (size_t)rexsim_host_out_bytes(s)));
    if (cfg->terrain == REXSIM_TERRAIN_RANDOM) {
        // vertical centring of each field: btHeightfieldTerrainShape local origin = (min+max)/2
        std::vector<float> h((size_t)65536), zo(cfg->nfields);
        for (int f = 0; f < cfg->nfields; f++) {
            CK(cudaMemcpy(h.data(), cfg->fields + (size_t)f * 65536, 65536 * sizeof(float), cudaMemcpyDeviceToHost));
            float lo = 1e30f, hi = -1e30f;
            for (float v : h) { lo = fminf(lo, v); hi = fmaxf(hi, v); }
            zo[f] = (float)(0.5 * ((double)lo + (double)hi));
        }
        CK(cudaMalloc(&s->d_zoff, cfg->nfields * sizeof(float)));
        CK(cudaMemcpy(s->d_zoff, zo.data(), cfg->nfields * sizeof(float), cudaMemcpyHostToDevice));
    }
    s->P.model = s->d_model; s->P.sf = s->d_sf; s->P.si = s->d_si;
    s->P.snap_f = s->d_snap_f; s->P.snap_i = s->d_snap_i; s->P.field_zoff = s->d_zoff;
    s->P.err = s->d_err; s->P.cmd_out = s->d_cmd;
    s->P.cost = s->d_cost; s->P.perm = nullptr;
    s->P.launched = s->launched;
    // settled reset snapshots: Rex.Reset's 100 + 0.5/dt holding sub-steps (rex.py:314-323), once per field
    for (int f = 0; f < s->nsnap; f++) {
        s->P.settle_snapshot = f;
        cudaError_t e = launch_settle(s->P, s->d_snap_f, s->d_snap_i, 0);
        if (e != cudaSuccess) return cuda_fail(e, "settle launch");
        s->launches++;
    }
    CK(cudaDeviceSynchronize());
    guard.s = nullptr;
    *out = s;
    return REXSIM_OK;
}

void rexsim_destroy(RexSim* s) {
    if (!s) return;
    cudaFree(s->d_model); cudaFree(s->d_sf); cudaFree(s->d_si); cudaFree(s->d_snap_f); cudaFree(s->d_snap_i);
    cudaFree(s->d_ring); cudaFree(s->d_snap_ring);
    cudaFree(s->d_zoff); cudaFree(s->d_err); cudaFree(s->d_cmd); cudaFree(s->d_act); cudaFree(s->d_out); cudaFree(s->d_perm); cudaFree(s->d_cost); cudaFree(s->d_hist);
    delete s;
}

int rexsim_step(RexSim* s, const float* actions, float* obs, float* reward, uint8_t* done, void* stream) {
    if (!s || !actions || !obs || !reward || !done) return fail(REXSIM_ERR_INVALID, "null argument");
    Params P = s->P;
    P.actions = actions; P.obs = obs; P.reward = reward; P.done = done;
    cudaError_t e = launch_step(P, (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(e, "step launch");
    s->launches++;
    return REXSIM_OK;
}

static size_t out_done_offset(const RexSim* s) { return ((size_t)s->P.N * s->O + s->P.N) * sizeof(float); }
static size_t out_err_offset(const RexSim* s) { return (out_done_offset(s) + (size_t)s->P.N + 3) & ~(size_t)3; }
int64_t rexsim_host_out_bytes(const RexSim* s) {
    if (!s) return 0;
    return (int64_t)(out_err_offset(s) + sizeof(int32_t) + 8);      // + 8 flag bytes the kernel sets directly on the zero-copy path
}
// true when p is page-locked host memory the device can address directly (UVA: same pointer value on both sides)
static bool device_can_address(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost && at.devicePointer == p;
}
int rexsim_step_host(RexSim* s, const float* h_actions, void* h_out, void* stream) {
    if (!s || !h_actions || !h_out) return fail(REXSIM_ERR_INVALID, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t N = s->P.N;
    Params P = s->P;
    // Small batches with pinned buffers: the kernel reads the actions from, and writes its results into, the host block
    // directly (zero-copy over PCIe) -- no DMA launches at all: the error bits travel as flag bytes the kernel sets in the
    // block, the device-side aggregate is cleared BEFORE the kernel.  Large batches stage through device buffers so the kernel
    // never waits on PCIe.
    const bool zero_copy = N <= 16384 && device_can_address(h_actions) && device_can_address(h_out);   // queried per call (~1 us)
    int32_t* h_err = reinterpret_cast<int32_t*>((char*)h_out + out_err_offset(s));
    uint8_t* h_flags = reinterpret_cast<uint8_t*>(h_err + 1);
    if (zero_copy) {
        memset(h_flags, 0, 8);
        CK(cudaMemsetAsync(s->d_err + N, 0, sizeof(int32_t), st));    // the aggregate is per step on the host path
        P.actions = h_actions;
        P.obs = (float*)h_out; P.reward = (float*)h_out + N * s->O; P.done = (uint8_t*)h_out + out_done_offset(s);
        P.err_host = h_flags;
    } else {
        CK(cudaMemcpyAsync(s->d_act, h_actions, N * s->A * sizeof(float), cudaMemcpyHostToDevice, st));
        P.actions = s->d_act;
        P.obs = (float*)s->d_out; P.reward = (float*)s->d_out + N * s->O; P.done = s->d_out + out_done_offset(s);
    }
    cudaError_t e = launch_step(P, st);
    if (e != cudaSuccess) return cuda_fail(e, "step launch");
    s->launches++;
    if (!zero_copy) {
        CK(cudaMemcpyAsync(h_out, s->d_out, out_err_offset(s), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(h_err, s->d_err + N, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        CK(cudaMemsetAsync(s->d_err + N, 0, sizeof(int32_t), st));
    }
    CK(cudaStreamSynchronize(st));
    if (zero_copy) {
        int32_t bits = 0;
        for (int b = 0; b < 8; b++) if (h_flags[b]) bits |= 1 << b;
        *h_err = bits;
    }
    return REXSIM_OK;
}

int rexsim_rebalance(RexSim* s, void* stream) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    cudaError_t e = launch_rebalance(s->d_cost, s->P.N, s->d_hist, s->d_perm, (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(e, "rebalance launch");
    s->launches += 3;
    s->P.perm = s->d_perm;              // steps enqueued after this call use the new grouping
    return REXSIM_OK;
}

int rexsim_reset(RexSim* s, const int32_t* idx, int32_t k, float* obs_out, void* stream) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    if (idx && k < 0) return fail(REXSIM_ERR_INVALID, "negative count");
    Params P = s->P;
    P.reset_idx = idx; P.reset_k = k;
    cudaError_t e = launch_reset(P, obs_out, (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(e, "reset launch");
    if (!idx || k > 0) s->launches++;
    return REXSIM_OK;
}

int rexsim_get_state(RexSim* s, float* out_f, int32_t* out_i, void* stream) {
    if (!s || !out_f || !out_i) return fail(REXSIM_ERR_INVALID, "null argument");
    cudaError_t e = launch_get_state(s->P, out_f, out_i, (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(e, "get_state launch");
    s->launches++;
    return REXSIM_OK;
}
int rexsim_set_state(RexSim* s, const float* in_f, void* stream) {
    if (!s || !in_f) return fail(REXSIM_ERR_INVALID, "null argument");
    cudaError_t e = launch_set_state(s->P, in_f, (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(e, "set_state launch");
    s->launches++;
    return REXSIM_OK;
}
int rexsim_state_buffers(RexSim* s, float** state_f, int32_t** state_i) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    if (state_f) *state_f = s->d_sf;
    if (state_i) *state_i = s->d_si;
    return REXSIM_OK;
}
int rexsim_history_buffer(RexSim* s, float** ring, int64_t* n_floats) {
    if (!s || !ring || !n_floats) return fail(REXSIM_ERR_INVALID, "null argument");
    *ring = s->d_ring;
    *n_floats = s->d_ring ? (int64_t)s->P.ring_depth * (s->P.cfg.num_motors == 18 ? HW_WORDS_ARM : HW_WORDS) * s->P.N : 0;
    return REXSIM_OK;
}
int rexsim_error_flags(RexSim* s, int32_t** err_flags) {
    if (!s || !err_flags) return fail(REXSIM_ERR_INVALID, "null argument");
    *err_flags = s->d_err;
    return REXSIM_OK;
}
int rexsim_clear_errors(RexSim* s, void* stream) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    CK(cudaMemsetAsync(s->d_err + s->P.N, 0, sizeof(int32_t), (cudaStream_t)stream));
    return REXSIM_OK;
}
int rexsim_last_command(RexSim* s, float** cmd) {
    if (!s || !cmd) return fail(REXSIM_ERR_INVALID, "null argument");
    *cmd = s->d_cmd;
    return REXSIM_OK;
}
int rexsim_solver_cost(RexSim* s, int32_t** cost) {
    if (!s || !cost) return fail(REXSIM_ERR_INVALID, "null argument");
    *cost = s->d_cost;
    return REXSIM_OK;
}
int64_t rexsim_launch_count(const RexSim* s) { return s ? s->launches : 0; }
int rexsim_last_step_build(const RexSim* s, int32_t* cta_threads, int32_t* ctas_per_sm, int32_t* sensor) {
    if (!s || !cta_threads || !ctas_per_sm || !sensor) return fail(REXSIM_ERR_INVALID, "null argument");
    *cta_threads = s->launched[0]; *ctas_per_sm = s->launched[1]; *sensor = s->launched[2];
    return REXSIM_OK;
}
uint32_t rexsim_rand_u32(uint64_t seed, uint32_t global_env, uint32_t reset_count, uint32_t slot) {
    return rand_u32(seed, global_env, reset_count, slot);
}

}  // extern "C"
