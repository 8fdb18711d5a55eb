// rexsim_capi.cu -- the C ABI declared in include/rexsim.h (plain pointers and sizes, no torch types).
#include "rexsim_kernel.cuh"
#include "rexsim_host.h"
#include <algorithm>
#include <array>
#include <cstring>
#include <cmath>
#include <tuple>
#include <vector>

namespace rexsim {
cudaError_t launch_step(const Params& P, cudaStream_t st);
cudaError_t launch_reset(const Params& P, float* obs_out, cudaStream_t st);
cudaError_t launch_settle(const Params& P, float* snap_f, int32_t* snap_i, int first, int npairs, cudaStream_t st);
cudaError_t launch_set_task_values(const Params& P, const int32_t* idx, int k, const float* values, uint32_t rows, cudaStream_t st);
cudaError_t launch_get_state(const Params& P, float* out_f, int32_t* out_i, cudaStream_t st);
cudaError_t launch_set_state(const Params& P, const float* in_f, cudaStream_t st);
cudaError_t launch_rebalance(const int32_t* cost, const uint8_t* group, int ngroups, int n, int32_t* hist, int32_t* perm,
                             cudaStream_t st);
cudaError_t launch_episode_summary(const Params& P, int clear, double* out, cudaStream_t st);
cudaError_t launch_render(const Params& P, const float* rt, const float* zrange, const int32_t* idx, int k, int W, int H,
                          float distance, float yaw_deg, float pitch_deg, uint8_t* rgb, cudaStream_t st, int* launches);
}  // namespace rexsim

using namespace rexsim;

// One launch of the step kernel per control step: the envs of one (terrain, mark, step unit, action_repeat, solver_iterations),
// which own slots perm[first, first + count); task, signal: the group's first env's, whose unit_of is the group's unit;
// motors: the mark's motor count, 12 or 18
struct LaunchGroup {
    int32_t terrain, motors, task, signal, repeat, iters, first, count;
    int32_t launched[3];               // step_kernel instance of the group's last launch: BLOCK, OCC, SENSOR
};
// One env's construction values, as the per-env setters give them (the config's otherwise)
struct EnvRecord {
    uint8_t terrain, task, signal;
    int32_t motors, repeat, iters;     // motor count (12 or 18), action_repeat, solver_iterations
    float kp, kd;                      // motor_kp, motor_kd
    double pd;                         // pd_latency
};
// One setting of the reset hold.  Rex.Reset clears the history and holds through ApplyAction (rex.py:303-323), so the settled
// state depends on the solver's cap, the pose held (hold_start), the robot held, the gains and the PD observation's latency.
struct HoldSetting {
    int32_t iters, start, motors;
    float kp, kd;
    double pd;
    bool operator==(const HoldSetting& o) const {
        return iters == o.iters && start == o.start && motors == o.motors && kp == o.kp && kd == o.kd && pd == o.pd;
    }
};

struct RexSim {
    Params P;                          // the handle's buffers are P's pointer fields, allocated from `mem`
    DeviceBuffers mem;
    float* zrange = nullptr;           // [nfields][2] lowest / highest centred height of each field (renderer)
    float* rt = nullptr;               // render table (rexsim_set_render_tables)
    uint8_t* ep_block = nullptr;       // episode statistics: the per-env block behind P.ep (episode_block_bytes)
    double* ep_summary = nullptr;      // [4] count, nonfinite, sum of scores, sum of lengths (rexsim_episode_summary)
    bool rt_set = false;
    int32_t* perm = nullptr;           // slot -> env, sorted by solver cost; P.perm points here after rexsim_rebalance (at once with
                                       // several launch groups: each group's envs in its slot range)
    int32_t* hist = nullptr;           // rexsim_rebalance's bins: 256 per launch group (group-major)
    float* act = nullptr;              // staging for rexsim_step_host
    uint8_t* out = nullptr;            // obs | reward | done (same layout as the host block)
    uint8_t* fin = nullptr;            // final obs | limit staging for rexsim_step_host_final (allocated on its first call)
    int A = 0;
    bool started = false;              // a reset or step has been enqueued: the frame wrappers can no longer be switched on
    std::vector<EnvRecord> env;        // each env's construction values (empty before the first per-env setter: the config's)
    std::vector<HoldSetting> holds;    // the hold settings of P.ev.gains / P.el.hold, in plan()'s order (empty: no table)
    bool values_on = false;            // rexsim_set_env_values was called
    double* latency = nullptr;         // [2][N] per-env control and pd latencies (rexsim_set_env_latencies; null: off)
    uint8_t* terrain = nullptr;        // [N] per-env terrains (rexsim_set_env_terrains; null: off); P.env_terrain points here
    float friction[2] = {0.f, 0.f};    // per-env terrains: friction of each terrain's envs, plane and heightfield
    int32_t* repeats = nullptr;        // [2][N] per-env action_repeat, solver_iterations (rexsim_set_env_repeats; null: off)
    uint8_t* tasks = nullptr;          // [2][N] per-env task, signal (rexsim_set_env_tasks; null: off); P.env_task points here
    uint8_t* marks = nullptr;          // [N] per-env marks, 1 arm / 0 base (rexsim_set_env_marks; null: off); P.env_mark points here
    float* snap_ring_base = nullptr;   // per-env marks with the sensor model: the base envs' snapshot ring, [settings * fields][D]
                                       // [HW_WORDS] (P.snap_ring is the arm's); the base launches read it as their P.snap_ring
    // The launch groups (empty: one launch over every slot with the config's values), terrain-major, plane first, then in
    // order of first appearance; group g owns slots perm[first_g, first_g + count_g).  `group` is each env's group, the key
    // rexsim_rebalance sorts on: the terrain bytes when the groups are exactly the two terrains, its own [N] bytes otherwise;
    // null for a batch of one group.
    std::vector<LaunchGroup> groups;
    const uint8_t* group = nullptr;
    uint8_t* group_bytes = nullptr;
    int64_t launches = 0;
    int32_t launched[3] = {0, 0, 0};   // step_kernel instance of the last step launch: BLOCK, OCC, SENSOR
};

// The handle's Params for the launches over one group's envs: its terrain with that terrain's friction, its mark (the base or
// arm build of the step and settle kernels), its task and signal (launch_step's unit, the auto-reset's draws, the settle's
// start pose), its sub-steps per control step and its PGS cap
static Params group_params(const RexSim* s, Params P, const LaunchGroup& g) {
    if (s->terrain) P.cfg.friction = s->friction[g.terrain];
    if (s->marks && g.motors == 12) P.snap_ring = s->snap_ring_base;
    P.cfg.terrain = g.terrain; P.cfg.num_motors = g.motors; P.cfg.task = g.task; P.cfg.signal = g.signal;
    P.cfg.action_repeat = g.repeat; P.cfg.solver_iterations = g.iters;
    return P;
}
// One control step of every env: one launch over every slot, or one launch per launch group over its slot range of the
// permutation, each choosing its build from its own size.  All on `st`, so a captured graph holds them all.
static int step_launches(RexSim* s, const Params& P, cudaStream_t st) {
    if (s->groups.empty()) return enqueue(s, launch_step(P, st), "step launch");
    for (LaunchGroup& g : s->groups) {
        Params G = group_params(s, P, g);
        G.perm = P.perm + g.first; G.nslots = g.count; G.launched = g.launched;
        if (int rc = enqueue(s, launch_step(G, st), "step launch")) return rc;
        memcpy(s->launched, g.launched, sizeof(s->launched));
    }
    return REXSIM_OK;
}

// byte offsets of the block rexsim_step_host fills: obs [N][O] at 0 | reward [N] | done [N] | pad to 4 | int32 error bits |
// 8 flag bytes the kernel sets directly on the zero-copy path
struct HostBlock { size_t reward, done, err, bytes; };
static HostBlock host_block(size_t N, size_t O) {
    HostBlock b;
    b.reward = N * O * sizeof(float);
    b.done = b.reward + N * sizeof(float);
    b.err = (b.done + N + 3) & ~(size_t)3;
    b.bytes = b.err + sizeof(int32_t) + 8;
    return b;
}

// Rex._GetDelayedObservation reads history[n] and history[n + 1], n = int(latency / dt), blended by a = (latency - n dt) / dt,
// in fp64 as the reference computes them
static Delay delay_terms(double latency, double dt) {
    Delay d;
    d.n = (int)(latency / dt);
    d.a = (float)((latency - d.n * dt) / dt);
    d.lat = (float)latency;
    return d;
}
// the sensor model a config asks for (all zero but `words` when it is off).  Per-env latencies run each env through this with
// the env's latencies in the config, so every env's terms are the scalar construction's.
struct SensorCfg { int on, depth; Delay ctl, pd; int words; };
static SensorCfg sensor_cfg(const RexSimConfig* c) {
    SensorCfg sc = {};
    sc.words = c->num_motors == 18 ? HW_WORDS_ARM : HW_WORDS;
    sc.on = c->control_latency > 0 || c->pd_latency > 0;
    for (int k = 0; k < 5; k++) sc.on = sc.on || c->noise_stdev[k] > 0;
    if (!sc.on) return sc;
    sc.ctl = delay_terms(c->control_latency, c->sim_dt_d);
    sc.pd = delay_terms(c->pd_latency, c->sim_dt_d);
    // rows read: n + 1 at most; once n + 1 reaches the deque's length (maxlen 100, rex.py:122) it reads the oldest row instead
    const int n = sc.ctl.n > sc.pd.n ? sc.ctl.n : sc.pd.n;
    sc.depth = n + 1 >= HIST_MAXLEN ? (int)HIST_MAXLEN : n + 2;
    return sc;
}

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
    if (c->num_motors == 18 && c->task == REXSIM_TASK_GALLOP)
        return fail(REXSIM_ERR_UNSUPPORTED, "mark='arm' is built for every task but gallop (its observation would carry the 18 motor angles)");
    if (c->action_repeat <= 0 || c->solver_iterations <= 0 || !(c->sim_dt_d > 0)) return fail(REXSIM_ERR_INVALID, "bad time stepping");
    // the step kernel switches a motor off once its overheat count c > floor(1 / sim_dt) (rex.py:601-608); c is a 10-bit
    // saturating field, so at floor(1 / sim_dt) >= 1023 the protection could never fire
    if ((uint32_t)(1.0 / c->sim_dt_d) >= 1023u)
        return fail(REXSIM_ERR_UNSUPPORTED, "sim_dt too small for the 10-bit overheat counter: needs floor(1 / sim_dt) <= 1022");
    if (c->terrain == REXSIM_TERRAIN_RANDOM && (c->nfields <= 0 || !c->fields)) return fail(REXSIM_ERR_INVALID, "random terrain needs a heightfield bank");
    if (c->terrain != REXSIM_TERRAIN_PLANE && c->terrain != REXSIM_TERRAIN_RANDOM) return fail(REXSIM_ERR_UNSUPPORTED, "terrain type");
    if (c->toe_npts <= 0 || c->toe_npts > REXSIM_MAX_TOE_PTS) return fail(REXSIM_ERR_MODEL, "toe_npts out of range");
    if (!(c->gait_clock_scale > 0)) return fail(REXSIM_ERR_INVALID, "gait_clock_scale must be positive (1 = simulation clock)");
    if (!(c->control_latency >= 0) || !(c->pd_latency >= 0)) return fail(REXSIM_ERR_INVALID, "latencies must be >= 0");
    for (int k = 0; k < 5; k++) if (!(c->noise_stdev[k] >= 0)) return fail(REXSIM_ERR_INVALID, "noise_stdev must be >= 0");
    if (c->episode_stats != 0 && c->episode_stats != 1) return fail(REXSIM_ERR_INVALID, "episode_stats must be 0 or 1");
    return REXSIM_OK;
}
int rexsim_history_depth(const RexSimConfig* c) { return c ? sensor_cfg(c).depth : 0; }
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
    Params& P = s->P;
    DeviceBuffers& mem = s->mem;
    memset(&P, 0, sizeof(Params));
    P.cfg = *cfg;
    P.cfg.sim_dt = (float)cfg->sim_dt_d;
    const size_t N = cfg->num_envs;
    P.N = cfg->num_envs;
    P.nslots = cfg->num_envs;
    {
        int dev = 0, sms = 132;
        CK(cudaGetDevice(&dev));
        CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        P.sm_count = sms;
    }
    P.snaps = snap_layout(cfg->terrain == REXSIM_TERRAIN_PLANE, cfg->terrain == REXSIM_TERRAIN_RANDOM, cfg->nfields);
    const size_t nsnap = P.snaps.per_setting;
    s->A = rexsim_action_dim(cfg->task, cfg->signal);
    P.out_dim = out_dim(cfg->task, cfg->num_motors, 0);
    // the kernels read these through pointers to const; create fills them
    float *model = nullptr, *snap_f = nullptr, *zoff = nullptr;
    int32_t* snap_i = nullptr;
    if (mem.zeroed(&model, mt_floats) || mem.zeroed(&P.sf, NF * N) || mem.zeroed(&P.si, NI * N) ||
        mem.zeroed(&snap_f, (size_t)NF * nsnap) || mem.zeroed(&snap_i, (size_t)NI * nsnap) ||
        mem.zeroed(&P.err, N + 1) ||                                    // [N] per-env bits + 1 word: OR of all
        mem.zeroed(&P.cmd_out, cfg->num_motors * N) || mem.zeroed(&P.cost, N) || mem.zeroed(&s->perm, N) ||
        mem.zeroed(&s->hist, 256) || mem.zeroed(&s->rt, REXSIM_RT_FLOATS) || mem.zeroed(&s->act, N * s->A) ||
        mem.zeroed(&s->out, host_block(N, P.out_dim).bytes))
        return REXSIM_ERR_CUDA;
    CK(cudaMemcpy(model, model_tables, mt_floats * sizeof(float), cudaMemcpyHostToDevice));
    const SensorCfg sc = sensor_cfg(cfg);
    if (sc.on) {
        P.sensor_on = 1;
        P.ring_depth = sc.depth;
        P.ctl = sc.ctl; P.pd = sc.pd;
        for (int k = 0; k < 5; k++) P.noise_sd[k] = (float)cfg->noise_stdev[k];
        if (mem.zeroed(&P.ring, (size_t)sc.depth * sc.words * N) || mem.zeroed(&P.snap_ring, nsnap * sc.depth * sc.words))
            return REXSIM_ERR_CUDA;
    }
    if (cfg->episode_stats) {
        if (mem.zeroed(&s->ep_block, episode_block_bytes(N)) || mem.zeroed(&s->ep_summary, 4)) return REXSIM_ERR_CUDA;
        EpisodeStats& E = P.ep;
        E.sum_score = reinterpret_cast<double*>(s->ep_block);
        E.sum_length = reinterpret_cast<int64_t*>(E.sum_score + N);
        E.score = reinterpret_cast<float*>(E.sum_length + N);
        E.length = reinterpret_cast<int32_t*>(E.score + N);
        E.count = E.length + N;
        E.nonfinite = E.count + N;
        // RexGymEnv._reward's objectives: turn, standup and poses override _reward and record none (turn_env.py:362-367,
        // standup_env.py:151-167, poses_env.py:256-258)
        if ((cfg->task == REXSIM_TASK_WALK || cfg->task == REXSIM_TASK_GALLOP) && mem.zeroed(&E.objectives, 4 * N))
            return REXSIM_ERR_CUDA;
    }
    if (cfg->terrain == REXSIM_TERRAIN_RANDOM) {
        // vertical centring of each field: btHeightfieldTerrainShape local origin = (min+max)/2
        std::vector<float> h((size_t)65536), zo(cfg->nfields), zr(2 * (size_t)cfg->nfields);
        for (int f = 0; f < cfg->nfields; f++) {
            CK(cudaMemcpy(h.data(), cfg->fields + (size_t)f * 65536, 65536 * sizeof(float), cudaMemcpyDeviceToHost));
            float lo = 1e30f, hi = -1e30f;
            for (float v : h) { lo = fminf(lo, v); hi = fmaxf(hi, v); }
            zo[f] = (float)(0.5 * ((double)lo + (double)hi));
            zr[2 * f] = lo - zo[f]; zr[2 * f + 1] = hi - zo[f];
        }
        if (mem.zeroed(&zoff, zo.size()) || mem.zeroed(&s->zrange, zr.size())) return REXSIM_ERR_CUDA;
        CK(cudaMemcpy(zoff, zo.data(), zo.size() * sizeof(float), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(s->zrange, zr.data(), zr.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    P.model = model; P.snap_f = snap_f; P.snap_i = snap_i; P.field_zoff = zoff;
    P.launched = s->launched;
    // settled reset snapshots: Rex.Reset's 100 + 0.5/dt holding sub-steps (rex.py:314-323), once per field
    if ((rc = enqueue(s, launch_settle(P, snap_f, snap_i, 0, 1, 0), "settle launch"))) return rc;
    CK(cudaDeviceSynchronize());
    guard.s = nullptr;
    *out = s;
    return REXSIM_OK;
}

void rexsim_destroy(RexSim* s) {
    if (!s) return;
    s->mem.release();
    delete s;
}

int rexsim_step(RexSim* s, const float* actions, float* obs, float* reward, uint8_t* done, void* stream) {
    if (!s || !actions || !obs || !reward || !done) return fail(REXSIM_ERR_INVALID, "null argument");
    Params P = s->P;
    P.actions = actions; P.obs = obs; P.reward = reward; P.done = done;
    s->started = true;
    return step_launches(s, P, (cudaStream_t)stream);
}
int rexsim_step_final(RexSim* s, const float* actions, float* obs, float* reward, uint8_t* done, float* final_obs,
                      uint8_t* limit, void* stream) {
    if (!s || !actions || !obs || !reward || !done) return fail(REXSIM_ERR_INVALID, "null argument");
    Params P = s->P;
    P.actions = actions; P.obs = obs; P.reward = reward; P.done = done; P.final_obs = final_obs; P.limit = limit;
    s->started = true;
    return step_launches(s, P, (cudaStream_t)stream);
}

// bytes of the block rexsim_step_host_final fills besides h_out: final obs [N][O] f32 | limit [N] u8
static size_t final_block_bytes(size_t N, size_t O) { return N * O * sizeof(float) + N; }
int64_t rexsim_host_final_bytes(const RexSim* s) { return s ? (int64_t)final_block_bytes(s->P.N, s->P.out_dim) : 0; }

int64_t rexsim_host_out_bytes(const RexSim* s) { return s ? (int64_t)host_block(s->P.N, s->P.out_dim).bytes : 0; }
int rexsim_out_dim(const RexSim* s) { return s ? s->P.out_dim : 0; }
// true when p is page-locked host memory the device can address directly (UVA: same pointer value on both sides)
static bool device_can_address(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost && at.devicePointer == p;
}
// rexsim_step_host, and rexsim_step_host_final when h_final is not null
static int step_host(RexSim* s, const float* h_actions, void* h_out, void* h_final, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const size_t N = s->P.N;
    const HostBlock hb = host_block(N, s->P.out_dim);
    const size_t fb = final_block_bytes(N, s->P.out_dim);
    Params P = s->P;
    // the staging block keeps the rows of envs that did not end from one call to the next, as the caller's block does on
    // the zero-copy path; its width is fixed once stepping has started (rexsim_set_frames)
    if (h_final && !s->fin && s->mem.zeroed(&s->fin, fb)) return REXSIM_ERR_CUDA;
    s->started = true;
    // Small batches with pinned buffers: the kernel reads the actions from, and writes its results into, the host block
    // directly (zero-copy over PCIe) -- no DMA launches at all: the error bits travel as flag bytes the kernel sets in the
    // block, the device-side aggregate is cleared BEFORE the kernel.  Large batches stage through device buffers so the kernel
    // never waits on PCIe.
    const bool zero_copy = N <= 16384 && device_can_address(h_actions) && device_can_address(h_out) &&
                           (!h_final || device_can_address(h_final));                     // queried per call (~1 us)
    int32_t* h_err = reinterpret_cast<int32_t*>((char*)h_out + hb.err);
    uint8_t* h_flags = reinterpret_cast<uint8_t*>(h_err + 1);
    if (zero_copy) {
        memset(h_flags, 0, 8);
        CK(cudaMemsetAsync(P.err + N, 0, sizeof(int32_t), st));       // the aggregate is per step on the host path
        P.actions = h_actions;
        P.err_host = h_flags;
    } else {
        CK(cudaMemcpyAsync(s->act, h_actions, N * s->A * sizeof(float), cudaMemcpyHostToDevice, st));
        P.actions = s->act;
    }
    uint8_t* block = zero_copy ? (uint8_t*)h_out : s->out;
    P.obs = (float*)block; P.reward = (float*)(block + hb.reward); P.done = block + hb.done;
    if (h_final) {
        uint8_t* fin = zero_copy ? (uint8_t*)h_final : s->fin;
        P.final_obs = (float*)fin; P.limit = fin + N * s->P.out_dim * sizeof(float);
    }
    if (int rc = step_launches(s, P, st)) return rc;
    if (!zero_copy) {
        CK(cudaMemcpyAsync(h_out, s->out, hb.err, cudaMemcpyDeviceToHost, st));
        if (h_final) CK(cudaMemcpyAsync(h_final, s->fin, fb, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(h_err, P.err + N, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        CK(cudaMemsetAsync(P.err + N, 0, sizeof(int32_t), st));
    }
    CK(cudaStreamSynchronize(st));
    if (zero_copy) {
        int32_t bits = 0;
        for (int b = 0; b < 8; b++) if (h_flags[b]) bits |= 1 << b;
        *h_err = bits;
    }
    return REXSIM_OK;
}
int rexsim_step_host(RexSim* s, const float* h_actions, void* h_out, void* stream) {
    if (!s || !h_actions || !h_out) return fail(REXSIM_ERR_INVALID, "null argument");
    return step_host(s, h_actions, h_out, nullptr, stream);
}
int rexsim_step_host_final(RexSim* s, const float* h_actions, void* h_out, void* h_final, void* stream) {
    if (!s || !h_actions || !h_out || !h_final) return fail(REXSIM_ERR_INVALID, "null argument");
    return step_host(s, h_actions, h_out, h_final, stream);
}

int rexsim_rebalance(RexSim* s, void* stream) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    const int rc = enqueue(s, launch_rebalance(s->P.cost, s->group, (int)s->groups.size(), s->P.N, s->hist, s->perm,
                                               (cudaStream_t)stream), "rebalance launch", 3);
    if (rc == REXSIM_OK) s->P.perm = s->perm;   // steps enqueued after this call use the new grouping
    return rc;
}

int rexsim_reset(RexSim* s, const int32_t* idx, int32_t k, float* obs_out, void* stream) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    if (idx && k < 0) return fail(REXSIM_ERR_INVALID, "negative count");
    Params P = s->P;
    P.reset_idx = idx; P.reset_k = k;
    s->started = true;
    if (s->marks) {
        // a batch of both marks: the base instance, on the base envs' snapshot ring, then the arm instance; each writes only
        // the envs of its own mark (P.env_mark)
        Params B = P;
        B.cfg.num_motors = 12; B.snap_ring = s->snap_ring_base;
        if (int rc = enqueue(s, launch_reset(B, obs_out, (cudaStream_t)stream), "reset launch", !idx || k > 0)) return rc;
    }
    return enqueue(s, launch_reset(P, obs_out, (cudaStream_t)stream), "reset launch", !idx || k > 0);
}

int rexsim_get_state(RexSim* s, float* out_f, int32_t* out_i, void* stream) {
    if (!s || !out_f || !out_i) return fail(REXSIM_ERR_INVALID, "null argument");
    return enqueue(s, launch_get_state(s->P, out_f, out_i, (cudaStream_t)stream), "get_state launch");
}
int rexsim_set_state(RexSim* s, const float* in_f, void* stream) {
    if (!s || !in_f) return fail(REXSIM_ERR_INVALID, "null argument");
    return enqueue(s, launch_set_state(s->P, in_f, (cudaStream_t)stream), "set_state launch");
}
int rexsim_state_buffers(RexSim* s, float** state_f, int32_t** state_i) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    if (state_f) *state_f = s->P.sf;
    if (state_i) *state_i = s->P.si;
    return REXSIM_OK;
}
int rexsim_history_buffer(RexSim* s, float** ring, int64_t* n_floats) {
    if (!s || !ring || !n_floats) return fail(REXSIM_ERR_INVALID, "null argument");
    const SensorCfg sc = sensor_cfg(&s->P.cfg);
    *ring = s->P.ring;
    *n_floats = (int64_t)s->P.ring_depth * sc.words * s->P.N;       // depth 0: the sensor model is off
    return REXSIM_OK;
}
int rexsim_error_flags(RexSim* s, int32_t** err_flags) {
    if (!s || !err_flags) return fail(REXSIM_ERR_INVALID, "null argument");
    *err_flags = s->P.err;
    return REXSIM_OK;
}
int rexsim_clear_errors(RexSim* s, void* stream) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    CK(cudaMemsetAsync(s->P.err + s->P.N, 0, sizeof(int32_t), (cudaStream_t)stream));
    return REXSIM_OK;
}
int rexsim_last_command(RexSim* s, float** cmd) {
    if (!s || !cmd) return fail(REXSIM_ERR_INVALID, "null argument");
    *cmd = s->P.cmd_out;
    return REXSIM_OK;
}
int rexsim_solver_cost(RexSim* s, int32_t** cost) {
    if (!s || !cost) return fail(REXSIM_ERR_INVALID, "null argument");
    *cost = s->P.cost;
    return REXSIM_OK;
}
int rexsim_set_render_tables(RexSim* s, const float* rt, int32_t n_floats) {
    if (!s || !rt) return fail(REXSIM_ERR_INVALID, "null argument");
    if (n_floats != REXSIM_RT_FLOATS) return fail(REXSIM_ERR_MODEL, "render table size mismatch");
    CK(cudaMemcpy(s->rt, rt, REXSIM_RT_FLOATS * sizeof(float), cudaMemcpyHostToDevice));
    s->rt_set = true;
    return REXSIM_OK;
}
int rexsim_render(RexSim* s, const int32_t* idx, int32_t k, int32_t width, int32_t height, float distance, float yaw_deg,
                  float pitch_deg, uint8_t* rgb, void* stream) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    if (k < 0) return fail(REXSIM_ERR_INVALID, "negative count");
    if (width < 1 || width > 4096 || height < 1 || height > 4096) return fail(REXSIM_ERR_INVALID, "image sides must be 1..4096");
    if (!s->rt_set) return fail(REXSIM_ERR_INVALID, "render tables not set (rexsim_set_render_tables)");
    if (k == 0) return REXSIM_OK;
    if (!idx || !rgb) return fail(REXSIM_ERR_INVALID, "null argument");
    int launches = 0;
    const cudaError_t e = launch_render(s->P, s->rt, s->zrange, idx, k, width, height, distance, yaw_deg, pitch_deg, rgb,
                                        (cudaStream_t)stream, &launches);
    return enqueue(s, e, "render launch", launches);
}
int rexsim_episode_buffers(RexSim* s, float** score, int32_t** length, float** objectives, double** summary, void** block,
                           int64_t* block_bytes) {
    if (!s || !score || !length || !objectives || !summary || !block || !block_bytes) return fail(REXSIM_ERR_INVALID, "null argument");
    if (!s->ep_block) return fail(REXSIM_ERR_INVALID, "episode statistics are off (RexSimConfig.episode_stats)");
    *score = s->P.ep.score; *length = s->P.ep.length; *objectives = s->P.ep.objectives; *summary = s->ep_summary;
    *block = s->ep_block; *block_bytes = (int64_t)episode_block_bytes(s->P.N);
    return REXSIM_OK;
}
int rexsim_episode_summary(RexSim* s, int32_t clear, void* stream) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    if (!s->ep_block) return fail(REXSIM_ERR_INVALID, "episode statistics are off (RexSimConfig.episode_stats)");
    return enqueue(s, launch_episode_summary(s->P, clear != 0, s->ep_summary, (cudaStream_t)stream), "episode summary launch");
}
int rexsim_set_frames(RexSim* s, const int32_t* past_indices, int32_t count, int32_t delta) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    if (s->started) return fail(REXSIM_ERR_INVALID, "frame wrappers must be set before the first reset or step");
    if (s->P.fr.ring || s->P.fr.last) return fail(REXSIM_ERR_INVALID, "frame wrappers are already set");
    if (delta != 0 && delta != 1) return fail(REXSIM_ERR_INVALID, "delta must be 0 or 1");
    if (count < 0 || count > FRAMES_MAX_INDICES) return fail(REXSIM_ERR_INVALID, "frame history takes 0 to 16 past indices");
    if (count > 0 && !past_indices) return fail(REXSIM_ERR_INVALID, "null past_indices");
    int capacity = 0;
    bool current = false;
    for (int k = 0; k < count; k++) {
        const int32_t i = past_indices[k];
        if (i < 0 || i > FRAMES_MAX_CAPACITY) return fail(REXSIM_ERR_INVALID, "past indices must lie in 0..64");
        capacity = i > capacity ? i : capacity;
        current = current || i == 0;
    }
    if (count > 0 && !current) return fail(REXSIM_ERR_INVALID, "Past indices should include 0 for the current frame.");
    if (count > 0 && capacity == 0) return fail(REXSIM_ERR_INVALID, "the largest past index must be positive (it is the ring's capacity)");
    if (count == 0 && !delta) return REXSIM_OK;
    Params& P = s->P;
    const size_t N = P.N;
    const int O = obs_dim(P.cfg.task, P.cfg.num_motors);
    if (delta && s->mem.zeroed(&P.fr.last, (size_t)O * N)) return REXSIM_ERR_CUDA;
    if (count > 0) {
        int32_t* index = nullptr;
        if (s->mem.zeroed(&P.fr.ring, (size_t)capacity * O * N) || s->mem.zeroed(&index, count)) return REXSIM_ERR_CUDA;
        CK(cudaMemcpy(index, past_indices, count * sizeof(int32_t), cudaMemcpyHostToDevice));
        P.fr.index = index; P.fr.capacity = capacity; P.fr.count = count;
    }
    P.out_dim = out_dim(P.cfg.task, P.cfg.num_motors, count);
    s->mem.drop(s->out);                                              // the host-path staging block takes the new width
    s->out = nullptr;
    if (s->mem.zeroed(&s->out, host_block(N, P.out_dim).bytes)) return REXSIM_ERR_CUDA;
    return REXSIM_OK;
}
int rexsim_frame_buffers(RexSim* s, float** ring, int64_t* ring_floats, float** last, int64_t* last_floats) {
    if (!s || !ring || !ring_floats || !last || !last_floats) return fail(REXSIM_ERR_INVALID, "null argument");
    const int64_t on = (int64_t)obs_dim(s->P.cfg.task, s->P.cfg.num_motors) * s->P.N;
    *ring = s->P.fr.ring; *ring_floats = s->P.fr.ring ? (int64_t)s->P.fr.capacity * on : 0;
    *last = s->P.fr.last; *last_floats = s->P.fr.last ? on : 0;
    return REXSIM_OK;
}
static const char* const c_value_keywords[REXSIM_VALUE_ROWS] = {
    "target_position", "backwards", "target_orient", "init_orient", "base_y", "base_z", "base_roll", "base_pitch", "base_yaw"};
static_assert(REXSIM_VALUE_POSE == 4 && REXSIM_VALUE_ROWS == REXSIM_VALUE_POSE + 5, "keyword table follows the row enum");
int rexsim_value_row(const char* keyword) {
    for (int r = 0; keyword && r < REXSIM_VALUE_ROWS; r++)
        if (!strcmp(keyword, c_value_keywords[r])) return r;
    return -1;
}
// The pose the reset hold of a (task, signal) ends in (settle_kernel): the IK stand, the open-loop stand (c_pose_stand_ol),
// standup's fold, or none (poses skips both holding phases)
enum { START_IK = 0, START_OL = 1, START_FOLD = 2, START_NONE = 3 };
static int32_t hold_start(int task, int signal) {
    return task == REXSIM_TASK_STANDUP ? START_FOLD : task == REXSIM_TASK_POSES ? START_NONE
         : signal == REXSIM_SIGNAL_OL ? START_OL : START_IK;
}
static EnvRecord config_record(const RexSimConfig& c) {
    return EnvRecord{(uint8_t)c.terrain, (uint8_t)c.task, (uint8_t)c.signal, c.num_motors, c.action_repeat, c.solver_iterations,
                     c.motor_kp, c.motor_kd, c.pd_latency};
}
// the handle's per-env records, or N copies of the config's values before the first per-env setter
static std::vector<EnvRecord> records(const RexSim* s) {
    return s->env.empty() ? std::vector<EnvRecord>(s->P.N, config_record(s->P.cfg)) : s->env;
}
static HoldSetting hold_of(const EnvRecord& r) { return HoldSetting{r.iters, hold_start(r.task, r.signal), r.motors, r.kp, r.kd, r.pd}; }

// What a record vector asks the step and the reset hold for.  groups: the launch groups (terrain, mark, step unit,
// action_repeat, solver_iterations), terrain-major, plane first, then in order of first appearance, with their slot ranges;
// group: each env's.  holds: the distinct hold settings, ordered by the env at which each one's PGS cap first appears, then
// its (cap, start), then its (cap, start, mark), then the setting itself, so that each cap's, (cap, start)'s and (cap, start,
// mark)'s settings are contiguous (settle_snapshots settles each (cap, start, mark) in one launch); hold: each env's.
struct Plan { std::vector<LaunchGroup> groups; std::vector<uint8_t> group; std::vector<HoldSetting> holds; std::vector<int32_t> hold; };
static int plan(const std::vector<EnvRecord>& r, Plan& p) {
    const size_t N = r.size();
    p.group.assign(N, 0);
    for (const int t : {REXSIM_TERRAIN_PLANE, REXSIM_TERRAIN_RANDOM})
        for (size_t e = 0; e < N; e++) {
            if (r[e].terrain != t) continue;
            size_t g = 0;
            while (g < p.groups.size() && !(p.groups[g].terrain == t && p.groups[g].motors == r[e].motors &&
                                             unit_of(p.groups[g].task, p.groups[g].signal) == unit_of(r[e].task, r[e].signal) &&
                                             p.groups[g].repeat == r[e].repeat && p.groups[g].iters == r[e].iters)) g++;
            if (g == p.groups.size()) {
                if ((int)g == REXSIM_MAX_LAUNCH_GROUPS)
                    return fail(REXSIM_ERR_INVALID, "more than 16 launch groups (terrain, mark, task unit, action_repeat, solver_iterations)");
                p.groups.push_back(LaunchGroup{t, r[e].motors, r[e].task, r[e].signal, r[e].repeat, r[e].iters, 0, 0, {0, 0, 0}});
            }
            p.groups[g].count++;
            p.group[e] = (uint8_t)g;
        }
    for (size_t g = 1; g < p.groups.size(); g++) p.groups[g].first = p.groups[g - 1].first + p.groups[g - 1].count;
    std::vector<HoldSetting> seen;                 // the distinct settings in order of first appearance
    std::vector<size_t> at;                        // the env each first appears at
    std::vector<int32_t> idx(N);
    for (size_t e = 0; e < N; e++) {
        const HoldSetting h = hold_of(r[e]);
        const size_t k = std::find(seen.begin(), seen.end(), h) - seen.begin();
        if (k == seen.size()) {
            if ((int)k == REXSIM_MAX_GAIN_PAIRS)
                return fail(REXSIM_ERR_INVALID, "more than 64 distinct reset-hold settings (mark, start pose, motor_kp, motor_kd, pd_latency, solver_iterations)");
            seen.push_back(h);
            at.push_back(e);
        }
        idx[e] = (int32_t)k;
    }
    // the sort key of setting k: the first appearance of its cap, (cap, start), (cap, start, mark) and of itself -- the first
    // setting sharing a prefix is the one that appears first
    auto prefix = [](const HoldSetting& h, int level) {
        return std::make_tuple(h.iters, level > 0 ? h.start : 0, level > 1 ? h.motors : 0);
    };
    std::vector<std::array<size_t, 4>> key(seen.size());
    for (size_t k = 0; k < seen.size(); k++) {
        for (int level = 0; level < 3; level++) {
            size_t j = 0;
            while (prefix(seen[j], level) != prefix(seen[k], level)) j++;
            key[k][level] = at[j];
        }
        key[k][3] = at[k];
    }
    std::vector<int32_t> order(seen.size()), rank(seen.size());
    for (size_t k = 0; k < seen.size(); k++) order[k] = (int32_t)k;
    std::sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return key[a] < key[b]; });
    p.holds.resize(seen.size());
    for (size_t i = 0; i < order.size(); i++) { p.holds[i] = seen[order[i]]; rank[order[i]] = (int32_t)i; }
    p.hold.resize(N);
    for (size_t e = 0; e < N; e++) p.hold[e] = rank[idx[e]];
    return REXSIM_OK;
}
// the launch groups a step launches: the table, or for a batch without one its single group over every slot
static std::vector<LaunchGroup> launch_groups(const RexSim* s) {
    if (!s->groups.empty()) return s->groups;
    const RexSimConfig& c = s->P.cfg;
    return {LaunchGroup{c.terrain, c.num_motors, c.task, c.signal, c.action_repeat, c.solver_iterations, 0, s->P.N,
                        {s->launched[0], s->launched[1], s->launched[2]}}};
}
// Install a plan's launch groups: put each group's envs in its slot range, in env order, and give rexsim_rebalance the group
// key.  Synchronous.
static int build_groups(RexSim* s, const Plan& p) {
    Params& P = s->P;
    const size_t N = P.N;
    const std::vector<LaunchGroup>& gs = p.groups;
    std::vector<int32_t> at(gs.size()), perm(N);
    for (size_t g = 0; g < gs.size(); g++) at[g] = gs[g].first;
    for (size_t e = 0; e < N; e++) perm[at[p.group[e]]++] = (int32_t)e;
    CK(cudaMemcpy(s->perm, perm.data(), N * sizeof(int32_t), cudaMemcpyHostToDevice));
    P.perm = s->perm;                          // the partition holds from the first step on
    s->mem.drop(s->group_bytes);
    s->group_bytes = nullptr;
    s->group = nullptr;
    if (gs.size() > 1) {
        int32_t* hist = nullptr;
        if (s->mem.zeroed(&hist, 256 * gs.size())) return REXSIM_ERR_CUDA;
        s->mem.drop(s->hist);
        s->hist = hist;
        if (gs.size() == 2 && gs[0].terrain == REXSIM_TERRAIN_PLANE && gs[1].terrain == REXSIM_TERRAIN_RANDOM) {
            s->group = s->terrain;             // the groups are exactly the two terrains: group g is terrain g
        } else {
            if (s->mem.zeroed(&s->group_bytes, N)) return REXSIM_ERR_CUDA;
            CK(cudaMemcpy(s->group_bytes, p.group.data(), N, cudaMemcpyHostToDevice));
            s->group = s->group_bytes;
        }
    }
    s->groups = gs;
    return REXSIM_OK;
}
// Install a plan's hold table: P.ev.pair, P.ev.gains and, with per-env latencies, P.el.hold.  Synchronous.
static int apply_holds(RexSim* s, const Plan& p) {
    Params& P = s->P;
    const size_t N = P.N, nh = p.holds.size();
    std::vector<float> gains(2 * nh);
    for (size_t h = 0; h < nh; h++) { gains[2 * h] = p.holds[h].kp; gains[2 * h + 1] = p.holds[h].kd; }
    int32_t* dpair = nullptr;
    float* dgains = nullptr;
    if (s->mem.zeroed(&dpair, N) || s->mem.zeroed(&dgains, gains.size())) return REXSIM_ERR_CUDA;
    CK(cudaMemcpy(dpair, p.hold.data(), N * sizeof(int32_t), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dgains, gains.data(), gains.size() * sizeof(float), cudaMemcpyHostToDevice));
    s->mem.drop((void*)P.ev.pair); s->mem.drop((void*)P.ev.gains);
    P.ev.pair = dpair; P.ev.gains = dgains;
    if (s->latency) {
        std::vector<Delay> hold(nh);
        for (size_t h = 0; h < nh; h++) hold[h] = delay_terms(p.holds[h].pd, P.cfg.sim_dt_d);
        Delay* dhold = nullptr;
        if (s->mem.zeroed(&dhold, nh)) return REXSIM_ERR_CUDA;
        CK(cudaMemcpy(dhold, hold.data(), nh * sizeof(Delay), cudaMemcpyHostToDevice));
        s->mem.drop((void*)P.el.hold);
        P.el.hold = dhold;
    }
    s->holds = p.holds;
    return REXSIM_OK;
}
// Run the reset hold again for every snapshot of the layout P.snaps, at the handle's hold settings (the config's one without a
// table), its sensor history rows at the handle's ring depth and row width: one launch per (terrain, PGS cap, start pose, mark)
// the launch groups hold, each at that terrain's friction, with that cap, with a task and signal of that start and with that
// mark's build, over all the (cap, start, mark)'s (setting, field) snapshots.  Synchronous.
static int settle_snapshots(RexSim* s) {
    Params& P = s->P;
    const std::vector<HoldSetting> holds = s->holds.empty() ? std::vector<HoldSetting>{hold_of(config_record(P.cfg))} : s->holds;
    const size_t nsettle = holds.size() * P.snaps.per_setting;
    float* snap_f = nullptr;
    int32_t* snap_i = nullptr;
    if (s->mem.zeroed(&snap_f, (size_t)NF * nsettle) || s->mem.zeroed(&snap_i, (size_t)NI * nsettle)) return REXSIM_ERR_CUDA;
    s->mem.drop((void*)P.snap_f); s->mem.drop((void*)P.snap_i);
    P.snap_f = snap_f; P.snap_i = snap_i;
    if (P.sensor_on) {
        s->mem.drop(P.snap_ring);
        P.snap_ring = nullptr;
        if (s->mem.zeroed(&P.snap_ring, nsettle * P.ring_depth * sensor_cfg(&P.cfg).words)) return REXSIM_ERR_CUDA;
        if (s->marks) {                        // the base envs' snapshots, at the base's row width
            s->mem.drop(s->snap_ring_base);
            s->snap_ring_base = nullptr;
            if (s->mem.zeroed(&s->snap_ring_base, nsettle * P.ring_depth * HW_WORDS)) return REXSIM_ERR_CUDA;
        }
    }
    const std::vector<LaunchGroup> gs = launch_groups(s);
    auto same_hold = [](const LaunchGroup& a, const LaunchGroup& b) {
        return a.terrain == b.terrain && a.iters == b.iters && hold_start(a.task, a.signal) == hold_start(b.task, b.signal) &&
               a.motors == b.motors;
    };
    for (size_t g = 0; g < gs.size(); g++) {
        bool settled = false;                  // an earlier group on the same terrain with the same cap, start and mark
        for (size_t h = 0; h < g; h++) settled = settled || same_hold(gs[h], gs[g]);
        if (settled) continue;
        const int32_t st = hold_start(gs[g].task, gs[g].signal);
        int first = -1, count = 0;             // the (cap, start, mark)'s settings are contiguous
        for (size_t h = 0; h < holds.size(); h++)
            if (holds[h].iters == gs[g].iters && holds[h].start == st && holds[h].motors == gs[g].motors) {
                first = first < 0 ? (int)h : first;
                count++;
            }
        const Params G = group_params(s, P, gs[g]);
        if (int rc = enqueue(s, launch_settle(G, snap_f, snap_i, first, count, 0), "settle launch")) return rc;
    }
    CK(cudaDeviceSynchronize());
    return REXSIM_OK;
}
// What a per-env setter installs of its plan, after its own device bytes (install)
enum { GROUPS = 1, HOLDS = 2, SETTLE = 4 };
// Take a setter's records, and install the parts `what` of their plan: the launch groups (build_groups), the hold table
// (apply_holds), and the reset hold run again (settle_snapshots).  Synchronous.
static int install(RexSim* s, std::vector<EnvRecord>&& rec, const Plan& p, int what) {
    s->env = std::move(rec);
    if (what & GROUPS) if (int rc = build_groups(s, p)) return rc;
    if (what & HOLDS) if (int rc = apply_holds(s, p)) return rc;
    return what & SETTLE ? settle_snapshots(s) : REXSIM_OK;
}
// The per-env setters' common refusals, each before anything changes: a null argument (null_msg), a handle already reset or
// stepped, and the setter's block already set (`set`)
static int setter_prelude(const RexSim* s, bool null_args, const char* null_msg, const char* what, bool set) {
    if (!s || null_args) return fail(REXSIM_ERR_INVALID, null_msg);
    char msg[96];
    if (s->started) {
        snprintf(msg, sizeof(msg), "per-env %s must be set before the first reset or step", what);
        return fail(REXSIM_ERR_INVALID, msg);
    }
    if (set) {
        snprintf(msg, sizeof(msg), "per-env %s are already set", what);
        return fail(REXSIM_ERR_INVALID, msg);
    }
    return REXSIM_OK;
}
int rexsim_set_env_values(RexSim* s, const float* values, const float* kp, const float* kd) {
    if (int rc = setter_prelude(s, !values || !kp != !kd, "null argument (kp and kd are given together or not at all)", "values",
                                s && s->values_on)) return rc;
    Params& P = s->P;
    const RexSimConfig& c = P.cfg;
    const size_t N = P.N;
    for (size_t e = 0; e < N; e++) {
        const float b = values[REXSIM_VALUE_BACKWARDS * N + e];
        if (b != -1.f && b != 0.f && b != 1.f) return fail(REXSIM_ERR_INVALID, "backwards values must be -1, 0 or 1");
    }
    std::vector<EnvRecord> rec = records(s);
    if (kp) {
        if (c.kp_lo != c.kp_hi || c.kd_lo != c.kd_hi)
            return fail(REXSIM_ERR_INVALID, "per-env gains cannot be combined with a motor_kp / motor_kd range");
        for (size_t e = 0; e < N; e++) {
            if (!(kp[e] >= 0.f) || !(kd[e] >= 0.f) || std::isinf(kp[e]) || std::isinf(kd[e]))
                return fail(REXSIM_ERR_INVALID, "gains must be finite and non-negative");
            rec[e].kp = kp[e]; rec[e].kd = kd[e];
        }
    }
    Plan p;
    if (int rc = plan(rec, p)) return rc;
    float* block = nullptr;
    if (s->mem.zeroed(&block, (size_t)REXSIM_VALUE_BLOCK_ROWS * N)) return REXSIM_ERR_CUDA;
    CK(cudaMemcpy(block, values, (size_t)REXSIM_VALUE_ROWS * N * sizeof(float), cudaMemcpyHostToDevice));
    // the running episodes (none yet) start with the constructor's direction
    CK(cudaMemcpy(block + (size_t)REXSIM_VALUE_EPISODE_BACKWARDS * N, values + (size_t)REXSIM_VALUE_BACKWARDS * N, N * sizeof(float),
                  cudaMemcpyHostToDevice));
    P.ev.values = block;
    s->values_on = true;
    // per-env gains: the reset hold again, once per (setting, field); without them a new table is the config's one setting,
    // whose snapshot rexsim_create settled
    return install(s, std::move(rec), p, kp ? HOLDS | SETTLE : P.ev.pair ? 0 : HOLDS);
}
int rexsim_set_env_latencies(RexSim* s, const double* control_latency, const double* pd_latency) {
    if (int rc = setter_prelude(s, false, "null handle", "latencies", s && s->latency)) return rc;
    Params& P = s->P;
    const RexSimConfig& c = P.cfg;
    const size_t N = P.N;
    std::vector<double> lat(2 * N);
    std::vector<EnvRecord> rec = records(s);
    for (size_t e = 0; e < N; e++) {
        lat[e] = control_latency ? control_latency[e] : c.control_latency;
        lat[N + e] = pd_latency ? pd_latency[e] : c.pd_latency;
        if (!(lat[e] >= 0) || !(lat[N + e] >= 0) || std::isinf(lat[e]) || std::isinf(lat[N + e]))
            return fail(REXSIM_ERR_INVALID, "latencies must be finite and non-negative");
        rec[e].pd = lat[N + e];
    }
    // each env's terms as a batch built with its latencies as scalars would have them; the ring keeps the deepest history
    std::vector<EnvDelay> env(N);
    int depth = 0, on = 0;
    for (size_t e = 0; e < N; e++) {
        RexSimConfig ce = c;
        ce.control_latency = lat[e]; ce.pd_latency = lat[N + e];
        const SensorCfg sc = sensor_cfg(&ce);
        env[e] = EnvDelay{sc.ctl, sc.pd, sc.on, 0};
        depth = sc.depth > depth ? sc.depth : depth;
        on = on || sc.on;
    }
    Plan p;
    if (int rc = plan(rec, p)) return rc;
    double* dlat = nullptr;
    EnvDelay* denv = nullptr;
    if (s->mem.zeroed(&dlat, 2 * N) || s->mem.zeroed(&denv, N)) return REXSIM_ERR_CUDA;
    CK(cudaMemcpy(dlat, lat.data(), 2 * N * sizeof(double), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(denv, env.data(), N * sizeof(EnvDelay), cudaMemcpyHostToDevice));
    s->latency = dlat;
    P.el.env = denv;
    if (on && depth != P.ring_depth) {          // a latency switches the sensor model on, exactly as a scalar one does
        s->mem.drop(P.ring);
        P.ring = nullptr;
        if (s->mem.zeroed(&P.ring, (size_t)depth * sensor_cfg(&c).words * N)) return REXSIM_ERR_CUDA;
        P.sensor_on = 1;
        P.ring_depth = depth;
        for (int k = 0; k < 5; k++) P.noise_sd[k] = (float)c.noise_stdev[k];
    }
    return install(s, std::move(rec), p, HOLDS | SETTLE);
}
int rexsim_env_latency_buffers(RexSim* s, double** latency, int32_t* depth) {
    if (!s || !latency || !depth) return fail(REXSIM_ERR_INVALID, "null argument");
    if (!s->latency) return fail(REXSIM_ERR_INVALID, "per-env latencies are off (rexsim_set_env_latencies)");
    *latency = s->latency; *depth = s->P.ring_depth;
    return REXSIM_OK;
}
int rexsim_set_env_terrains(RexSim* s, const int32_t* terrain, float plane_friction) {
    if (int rc = setter_prelude(s, !terrain, "null argument", "terrains", s && s->terrain)) return rc;
    Params& P = s->P;
    if (P.cfg.terrain != REXSIM_TERRAIN_RANDOM)
        return fail(REXSIM_ERR_INVALID, "per-env terrains need a handle created on the random terrain (its heightfield bank)");
    if (!(plane_friction >= 0.f) || std::isinf(plane_friction)) return fail(REXSIM_ERR_INVALID, "plane friction must be finite and non-negative");
    const size_t N = P.N;
    std::vector<EnvRecord> rec = records(s);
    std::vector<uint8_t> bytes(N);
    size_t nplane = 0;
    for (size_t e = 0; e < N; e++) {
        if (terrain[e] != REXSIM_TERRAIN_PLANE && terrain[e] != REXSIM_TERRAIN_RANDOM)
            return fail(REXSIM_ERR_INVALID, "terrain entries must be REXSIM_TERRAIN_PLANE or REXSIM_TERRAIN_RANDOM");
        bytes[e] = rec[e].terrain = (uint8_t)terrain[e];
        nplane += terrain[e] == REXSIM_TERRAIN_PLANE;
    }
    Plan p;
    if (int rc = plan(rec, p)) return rc;
    uint8_t* dterrain = nullptr;
    if (s->mem.zeroed(&dterrain, N)) return REXSIM_ERR_CUDA;
    CK(cudaMemcpy(dterrain, bytes.data(), N, cudaMemcpyHostToDevice));
    s->terrain = dterrain;
    s->friction[REXSIM_TERRAIN_PLANE] = plane_friction; s->friction[REXSIM_TERRAIN_RANDOM] = P.cfg.friction;
    P.env_terrain = dterrain;
    P.snaps = snap_layout(nplane > 0, nplane < N, P.cfg.nfields);
    return install(s, std::move(rec), p, GROUPS | SETTLE);     // the terrain is no part of a hold setting
}
int rexsim_env_terrain_buffers(RexSim* s, uint8_t** terrain, int32_t* nplane) {
    if (!s || !terrain || !nplane) return fail(REXSIM_ERR_INVALID, "null argument");
    if (!s->terrain) return fail(REXSIM_ERR_INVALID, "per-env terrains are off (rexsim_set_env_terrains)");
    *terrain = s->terrain;
    *nplane = 0;
    for (const LaunchGroup& g : s->groups) if (g.terrain == REXSIM_TERRAIN_PLANE) *nplane += g.count;
    return REXSIM_OK;
}
int rexsim_set_env_repeats(RexSim* s, const int32_t* action_repeat, const int32_t* solver_iterations) {
    if (int rc = setter_prelude(s, false, "null handle", "repeats", s && s->repeats)) return rc;
    Params& P = s->P;
    const RexSimConfig& c = P.cfg;
    const size_t N = P.N;
    std::vector<EnvRecord> rec = records(s);
    std::vector<int32_t> rep(N), iters(N);
    std::vector<std::pair<int32_t, int32_t>> pairs;
    for (size_t e = 0; e < N; e++) {
        rep[e] = action_repeat ? action_repeat[e] : c.action_repeat;
        iters[e] = solver_iterations ? solver_iterations[e] : c.solver_iterations;
        if (rep[e] <= 0 || iters[e] <= 0) return fail(REXSIM_ERR_INVALID, "action_repeat and solver_iterations must be positive");
        if (std::find(pairs.begin(), pairs.end(), std::make_pair(rep[e], iters[e])) == pairs.end()) {
            if ((int)pairs.size() == REXSIM_MAX_REPEAT_PAIRS)
                return fail(REXSIM_ERR_INVALID, "more than 8 distinct (action_repeat, solver_iterations) pairs");
            pairs.push_back(std::make_pair(rep[e], iters[e]));
        }
        rec[e].repeat = rep[e]; rec[e].iters = iters[e];
    }
    Plan p;
    if (int rc = plan(rec, p)) return rc;
    int32_t* d = nullptr;
    if (s->mem.zeroed(&d, 2 * N)) return REXSIM_ERR_CUDA;
    CK(cudaMemcpy(d, rep.data(), N * sizeof(int32_t), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d + N, iters.data(), N * sizeof(int32_t), cudaMemcpyHostToDevice));
    s->repeats = d;
    return install(s, std::move(rec), p, GROUPS | HOLDS | SETTLE);
}
int rexsim_env_repeat_buffers(RexSim* s, int32_t** repeats) {
    if (!s || !repeats) return fail(REXSIM_ERR_INVALID, "null argument");
    if (!s->repeats) return fail(REXSIM_ERR_INVALID, "per-env repeats are off (rexsim_set_env_repeats)");
    *repeats = s->repeats;
    return REXSIM_OK;
}
int rexsim_set_env_tasks(RexSim* s, const int32_t* task, const int32_t* signal) {
    if (int rc = setter_prelude(s, !task || !signal, "null argument", "tasks", s && s->tasks)) return rc;
    Params& P = s->P;
    const RexSimConfig& c = P.cfg;
    const size_t N = P.N;
    // the reference's BatchEnv refuses envs whose spaces differ (batch_env.py:36-43): the widths always, the raw action bound
    // unless ClipAction and RangeNormalize replace both boxes (the observation bounds depend on the time step alone)
    const TaskShape own = task_shape(c.task);
    std::vector<EnvRecord> rec = records(s);
    std::vector<uint8_t> tk(N), sg(N);
    bool objectives = false;
    for (size_t e = 0; e < N; e++) {
        const int32_t k = task[e], g = signal[e];
        if (k < REXSIM_TASK_WALK || k > REXSIM_TASK_POSES || (g != REXSIM_SIGNAL_IK && g != REXSIM_SIGNAL_OL))
            return fail(REXSIM_ERR_INVALID, "task entries must be REXSIM_TASK_* and signal entries REXSIM_SIGNAL_*");
        if (k == REXSIM_TASK_GALLOP && c.num_motors == 18)
            return fail(REXSIM_ERR_INVALID, "mark='arm' is built for every task but gallop");
        if (rexsim_action_dim(k, g) != s->A || obs_dim(k, c.num_motors) != obs_dim(c.task, c.num_motors))
            return fail(REXSIM_ERR_INVALID, "All environments must use the same observation space (action or observation width differs)");
        if (!c.normalize && task_shape(k).bound[g] != own.bound[c.signal])
            return fail(REXSIM_ERR_INVALID, "All environments must use the same observation space (raw action bound differs)");
        tk[e] = rec[e].task = (uint8_t)k; sg[e] = rec[e].signal = (uint8_t)g;
        objectives = objectives || k == REXSIM_TASK_WALK || k == REXSIM_TASK_GALLOP;
    }
    Plan p;
    if (int rc = plan(rec, p)) return rc;
    uint8_t* d = nullptr;
    if (s->mem.zeroed(&d, 2 * N)) return REXSIM_ERR_CUDA;
    CK(cudaMemcpy(d, tk.data(), N, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d + N, sg.data(), N, cudaMemcpyHostToDevice));
    s->tasks = d;
    P.env_task = d;
    if (s->ep_block && objectives) {
        // walk and gallop record the objectives of every step; the other envs' columns are NaN and stay NaN
        std::vector<float> o(4 * N, 0.f);
        for (size_t e = 0; e < N; e++)
            if (tk[e] != REXSIM_TASK_WALK && tk[e] != REXSIM_TASK_GALLOP)
                for (int r = 0; r < 4; r++) o[r * N + e] = NAN;
        if (!P.ep.objectives && s->mem.zeroed(&P.ep.objectives, 4 * N)) return REXSIM_ERR_CUDA;
        CK(cudaMemcpy(P.ep.objectives, o.data(), 4 * N * sizeof(float), cudaMemcpyHostToDevice));
    }
    return install(s, std::move(rec), p, GROUPS | HOLDS | SETTLE);
}
int rexsim_env_task_buffers(RexSim* s, uint8_t** task) {
    if (!s || !task) return fail(REXSIM_ERR_INVALID, "null argument");
    if (!s->tasks) return fail(REXSIM_ERR_INVALID, "per-env tasks are off (rexsim_set_env_tasks)");
    *task = s->tasks;
    return REXSIM_OK;
}
int rexsim_launch_group_task(const RexSim* s, int32_t g, int32_t* task, int32_t* signal) {
    if (!s || !task || !signal) return fail(REXSIM_ERR_INVALID, "null argument");
    const std::vector<LaunchGroup> gs = launch_groups(s);
    if (g < 0 || g >= (int32_t)gs.size()) return fail(REXSIM_ERR_INVALID, "no such launch group");
    *task = gs[g].task; *signal = gs[g].signal;
    return REXSIM_OK;
}
int rexsim_set_env_marks(RexSim* s, const int32_t* num_motors) {
    if (int rc = setter_prelude(s, !num_motors, "null argument", "marks", s && s->marks)) return rc;
    Params& P = s->P;
    const size_t N = P.N;
    // the arm's model table starts with the base's (REXSIM_MT_FLOATS), its render table draws the base's shapes, its ring rows
    // hold the base's words first: a handle built for the arm serves base envs, not the other way round
    if (P.cfg.num_motors != 18) return fail(REXSIM_ERR_INVALID, "per-env marks need a handle created with the arm (num_motors 18)");
    std::vector<EnvRecord> rec = records(s);
    std::vector<uint8_t> bytes(N);
    for (size_t e = 0; e < N; e++) {
        if (num_motors[e] != 12 && num_motors[e] != 18) return fail(REXSIM_ERR_INVALID, "mark entries must be 12 (base) or 18 (arm)");
        if (num_motors[e] == 18 && rec[e].task == REXSIM_TASK_GALLOP)
            return fail(REXSIM_ERR_INVALID, "mark='arm' is built for every task but gallop");
        rec[e].motors = num_motors[e];
        bytes[e] = (uint8_t)(num_motors[e] == 18);
    }
    Plan p;
    if (int rc = plan(rec, p)) return rc;
    uint8_t* d = nullptr;
    if (s->mem.zeroed(&d, N)) return REXSIM_ERR_CUDA;
    CK(cudaMemcpy(d, bytes.data(), N, cudaMemcpyHostToDevice));
    // rows 12..17 of the [18][N] command block (still zero: nothing has stepped): NaN in a base env's column, which the base
    // build never writes
    std::vector<float> arm_rows(6 * N, 0.f);
    for (size_t e = 0; e < N; e++)
        if (!bytes[e]) for (int j = 0; j < 6; j++) arm_rows[j * N + e] = NAN;
    CK(cudaMemcpy(P.cmd_out + 12 * N, arm_rows.data(), 6 * N * sizeof(float), cudaMemcpyHostToDevice));
    s->marks = d;
    P.env_mark = d;
    return install(s, std::move(rec), p, GROUPS | HOLDS | SETTLE);
}
int rexsim_env_mark_buffers(RexSim* s, uint8_t** mark) {
    if (!s || !mark) return fail(REXSIM_ERR_INVALID, "null argument");
    if (!s->marks) return fail(REXSIM_ERR_INVALID, "per-env marks are off (rexsim_set_env_marks)");
    *mark = s->marks;
    return REXSIM_OK;
}
int rexsim_launch_group_mark(const RexSim* s, int32_t g, int32_t* num_motors) {
    if (!s || !num_motors) return fail(REXSIM_ERR_INVALID, "null argument");
    const std::vector<LaunchGroup> gs = launch_groups(s);
    if (g < 0 || g >= (int32_t)gs.size()) return fail(REXSIM_ERR_INVALID, "no such launch group");
    *num_motors = gs[g].motors;
    return REXSIM_OK;
}
int rexsim_launch_groups(const RexSim* s) { return s ? (int)launch_groups(s).size() : 0; }
int rexsim_launch_group(const RexSim* s, int32_t g, int32_t* info) {
    if (!s || !info) return fail(REXSIM_ERR_INVALID, "null argument");
    const std::vector<LaunchGroup> gs = launch_groups(s);
    if (g < 0 || g >= (int32_t)gs.size()) return fail(REXSIM_ERR_INVALID, "no such launch group");
    const LaunchGroup& G = gs[g];
    const int32_t w[REXSIM_GROUP_WORDS] = {G.terrain, G.repeat, G.iters, G.first, G.count, G.launched[0], G.launched[1], G.launched[2]};
    memcpy(info, w, sizeof(w));
    return REXSIM_OK;
}
int rexsim_slot_buffers(RexSim* s, int32_t** perm, uint8_t** group) {
    if (!s || !perm || !group) return fail(REXSIM_ERR_INVALID, "null argument");
    *perm = const_cast<int32_t*>(s->P.perm); *group = const_cast<uint8_t*>(s->group);
    return REXSIM_OK;
}
int rexsim_last_terrain_build(const RexSim* s, int32_t terrain, int32_t* cta_threads, int32_t* ctas_per_sm, int32_t* sensor) {
    if (!s || !cta_threads || !ctas_per_sm || !sensor) return fail(REXSIM_ERR_INVALID, "null argument");
    if (terrain != REXSIM_TERRAIN_PLANE && terrain != REXSIM_TERRAIN_RANDOM) return fail(REXSIM_ERR_INVALID, "terrain type");
    int32_t b[3] = {0, 0, 0};
    for (const LaunchGroup& g : launch_groups(s)) if (g.terrain == terrain) memcpy(b, g.launched, sizeof(b));
    *cta_threads = b[0]; *ctas_per_sm = b[1]; *sensor = b[2];
    return REXSIM_OK;
}
int rexsim_set_task_values(RexSim* s, const int32_t* idx, int32_t k, const float* values, uint32_t rows, void* stream) {
    if (!s) return fail(REXSIM_ERR_INVALID, "null handle");
    if (!s->values_on) return fail(REXSIM_ERR_INVALID, "per-env values are off (rexsim_set_env_values)");
    if (rows >> REXSIM_VALUE_ROWS) return fail(REXSIM_ERR_INVALID, "rows names a row past REXSIM_VALUE_ROWS");
    if (idx && k < 0) return fail(REXSIM_ERR_INVALID, "negative count");
    if (!idx) k = s->P.N;
    if (k == 0 || rows == 0) return REXSIM_OK;
    if (!values) return fail(REXSIM_ERR_INVALID, "null values");
    return enqueue(s, launch_set_task_values(s->P, idx, k, values, rows, (cudaStream_t)stream), "set_task_values launch");
}
int rexsim_env_value_buffers(RexSim* s, float** values, int32_t** pair, float** gains, int32_t* npairs) {
    if (!s || !values || !pair || !gains || !npairs) return fail(REXSIM_ERR_INVALID, "null argument");
    if (!s->values_on) return fail(REXSIM_ERR_INVALID, "per-env values are off (rexsim_set_env_values)");
    *values = s->P.ev.values; *pair = const_cast<int32_t*>(s->P.ev.pair); *gains = const_cast<float*>(s->P.ev.gains);
    *npairs = (int32_t)s->holds.size();
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
