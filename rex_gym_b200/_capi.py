"""ctypes binding of the C ABI in include/rexsim.h.  There is NO CPU fallback: if librexsim.so is
missing or CUDA is unavailable the product path raises."""
import ctypes as C
import os

from . import build as _build

HERE = os.path.dirname(os.path.abspath(__file__))


class RexSimConfig(C.Structure):
    _fields_ = [
        ("num_envs", C.c_int32), ("task", C.c_int32), ("signal", C.c_int32), ("terrain", C.c_int32),
        ("num_motors", C.c_int32), ("action_repeat", C.c_int32), ("solver_iterations", C.c_int32),
        ("sim_dt", C.c_float), ("sim_dt_d", C.c_double),
        ("motor_kp", C.c_float), ("motor_kd", C.c_float),
        ("kp_lo", C.c_float), ("kp_hi", C.c_float), ("kd_lo", C.c_float), ("kd_hi", C.c_float),
        ("target_position", C.c_float), ("backwards", C.c_int32),
        ("target_orient", C.c_float), ("init_orient", C.c_float),
        ("w_distance", C.c_float), ("w_energy", C.c_float), ("w_drift", C.c_float), ("w_shake", C.c_float),
        ("normalize", C.c_int32), ("max_episode_steps", C.c_int32), ("auto_reset", C.c_int32),
        ("seed", C.c_uint64), ("nfields", C.c_int32), ("fields", C.c_void_p),
        ("friction", C.c_float), ("residual_threshold", C.c_float), ("erp_contact", C.c_float), ("erp_joint", C.c_float),
        ("toe_npts", C.c_int32), ("toe_margin", C.c_float),
        ("contact_breaking", C.c_float), ("link_damping", C.c_float), ("max_coordinate_velocity", C.c_float), ("env_offset", C.c_int32),
        ("gait_clock_scale", C.c_double), ("pose_values", C.c_float * 5),
        ("control_latency", C.c_double), ("pd_latency", C.c_double), ("noise_stdev", C.c_double * 5),
    ]


class RexAgentConfig(C.Structure):
    _fields_ = [("obs_dim", C.c_int32), ("action_dim", C.c_int32), ("hidden1", C.c_int32), ("hidden2", C.c_int32),
                ("observ_clip", C.c_float), ("reward_clip", C.c_float)]


AGENT_EXPORTS = ["rexagent_policy_floats", "rexagent_value_floats", "rexagent_create", "rexagent_destroy", "rexagent_set_precision", "rexagent_set_params",
                 "rexagent_get_params", "rexagent_params_buffer", "rexagent_state_buffers", "rexagent_set_filters", "rexagent_get_filters",
                 "rexagent_perform", "rexagent_experience", "rexagent_experience_partial", "rexagent_experience_finalize", "rexagent_transform_reward", "rexagent_discounted_return",
                 "rexagent_lambda_advantage", "rexagent_gae_segments", "rexagent_launch_count"]

EXPORTS = ["rexsim_obs_dim", "rexsim_action_dim", "rexsim_state_words", "rexsim_create", "rexsim_destroy",
           "rexsim_step", "rexsim_step_host", "rexsim_host_out_bytes", "rexsim_rebalance", "rexsim_reset", "rexsim_get_state", "rexsim_set_state", "rexsim_state_buffers",
           "rexsim_error_flags", "rexsim_clear_errors", "rexsim_last_command", "rexsim_solver_cost", "rexsim_launch_count", "rexsim_last_step_build", "rexsim_last_error", "rexsim_rand_u32",
           "rexsim_noise", "rexsim_history_depth", "rexsim_history_buffer"]

_LIB = None


def lib_path():
    # REXSIM_LIB: developer override to A/B kernels built with other flags (must still be an in-tree build)
    return os.environ.get("REXSIM_LIB") or os.path.join(HERE, "librexsim.so")


def load():
    """Load librexsim.so (building it in-tree if the sources are newer).  Raises if impossible."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.environ.get("REXSIM_LIB") and _build.needs_build():
        _build.build()
    L = C.CDLL(lib_path())
    L.rexsim_obs_dim.argtypes = [C.c_int32, C.c_int32]
    L.rexsim_action_dim.argtypes = [C.c_int32, C.c_int32]
    L.rexsim_state_words.argtypes = [C.POINTER(RexSimConfig), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.rexsim_create.argtypes = [C.POINTER(RexSimConfig), C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]
    L.rexsim_destroy.argtypes = [C.c_void_p]
    L.rexsim_destroy.restype = None
    L.rexsim_step.argtypes = [C.c_void_p] * 6
    L.rexsim_step_host.argtypes = [C.c_void_p] * 4
    L.rexsim_host_out_bytes.argtypes = [C.c_void_p]
    L.rexsim_host_out_bytes.restype = C.c_int64
    L.rexsim_rebalance.argtypes = [C.c_void_p, C.c_void_p]
    L.rexsim_reset.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    L.rexsim_get_state.argtypes = [C.c_void_p] * 4
    L.rexsim_set_state.argtypes = [C.c_void_p] * 3
    L.rexsim_state_buffers.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    L.rexsim_error_flags.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    L.rexsim_clear_errors.argtypes = [C.c_void_p, C.c_void_p]
    L.rexsim_last_command.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    L.rexsim_solver_cost.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    L.rexsim_launch_count.argtypes = [C.c_void_p]
    L.rexsim_launch_count.restype = C.c_int64
    L.rexsim_last_step_build.argtypes = [C.c_void_p] + [C.POINTER(C.c_int32)] * 3
    L.rexsim_last_error.restype = C.c_char_p
    L.rexsim_rand_u32.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32]
    L.rexsim_rand_u32.restype = C.c_uint32
    L.rexsim_noise.argtypes = [C.c_uint64] + [C.c_uint32] * 5
    L.rexsim_noise.restype = C.c_float
    L.rexsim_history_depth.argtypes = [C.POINTER(RexSimConfig)]
    L.rexsim_history_buffer.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
    # include/rexsim_agent.h
    cfgp = C.POINTER(RexAgentConfig)
    L.rexagent_policy_floats.argtypes = [cfgp]; L.rexagent_policy_floats.restype = C.c_int64
    L.rexagent_value_floats.argtypes = [cfgp]; L.rexagent_value_floats.restype = C.c_int64
    L.rexagent_create.argtypes = [cfgp, C.POINTER(C.c_void_p)]
    L.rexagent_destroy.argtypes = [C.c_void_p]; L.rexagent_destroy.restype = None
    L.rexagent_set_precision.argtypes = [C.c_void_p, C.c_int32]
    L.rexagent_set_params.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    L.rexagent_get_params.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    L.rexagent_params_buffer.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    L.rexagent_state_buffers.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    L.rexagent_set_filters.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_float]
    L.rexagent_get_filters.argtypes = [C.c_void_p] * 5
    L.rexagent_perform.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_uint64, C.c_uint32, C.c_uint32] + [C.c_void_p] * 6
    L.rexagent_experience.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    L.rexagent_experience_partial.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    L.rexagent_experience_finalize.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.rexagent_transform_reward.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    L.rexagent_discounted_return.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int64, C.c_float, C.c_void_p, C.c_void_p]
    L.rexagent_lambda_advantage.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int64, C.c_float, C.c_void_p, C.c_void_p]
    L.rexagent_gae_segments.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    L.rexagent_launch_count.argtypes = [C.c_void_p]; L.rexagent_launch_count.restype = C.c_int64
    _LIB = L
    return L


def check(rc):
    if rc == 0:
        return
    msg = load().rexsim_last_error().decode()
    if rc in (-1, -2, -4):
        raise ValueError(f"rexsim: {msg} (status {rc})")
    raise RuntimeError(f"rexsim: {msg} (status {rc})")
