"""ctypes binding of the C ABI in include/rexsim.h.  There is NO CPU fallback: if librexsim.so is
missing or CUDA is unavailable the product path raises."""
import ctypes as C
import os

import torch

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
        ("episode_stats", C.c_int32),
    ]


class RexAgentConfig(C.Structure):
    _fields_ = [("obs_dim", C.c_int32), ("action_dim", C.c_int32), ("hidden1", C.c_int32), ("hidden2", C.c_int32),
                ("observ_clip", C.c_float), ("reward_clip", C.c_float)]


class RexRnnConfig(C.Structure):
    _fields_ = [("kind", C.c_int32), ("hidden1", C.c_int32), ("cell", C.c_int32), ("num_envs", C.c_int32)]


REXRNN_GRU, REXRNN_LINEAR = 0, 1

_i32, _i64, _u32, _u64, _f32, _ptr = C.c_int32, C.c_int64, C.c_uint32, C.c_uint64, C.c_float, C.c_void_p
_out, _sim_cfg, _agent_cfg = C.POINTER, C.POINTER(RexSimConfig), C.POINTER(RexAgentConfig)
_rnn_cfg = C.POINTER(RexRnnConfig)

# name: (restype, argtypes) of every function of include/rexsim.h, include/rexsim_agent.h and include/rexsim_recurrent.h.  load() declares exactly these,
# and the export lists below are its keys: a function ctypes has no signature for would get C ints and truncated pointers.
SIGNATURES = {
    "rexsim_obs_dim": (C.c_int, [_i32, _i32]),
    "rexsim_action_dim": (C.c_int, [_i32, _i32]),
    "rexsim_state_words": (C.c_int, [_sim_cfg, _out(_i32), _out(_i32)]),
    "rexsim_create": (C.c_int, [_sim_cfg, _ptr, _i32, _out(_ptr)]),
    "rexsim_destroy": (None, [_ptr]),
    "rexsim_step": (C.c_int, [_ptr] * 6),
    "rexsim_step_host": (C.c_int, [_ptr] * 4),
    "rexsim_host_out_bytes": (_i64, [_ptr]),
    "rexsim_step_final": (C.c_int, [_ptr] * 8),
    "rexsim_host_final_bytes": (_i64, [_ptr]),
    "rexsim_step_host_final": (C.c_int, [_ptr] * 5),
    "rexsim_rebalance": (C.c_int, [_ptr, _ptr]),
    "rexsim_reset": (C.c_int, [_ptr, _ptr, _i32, _ptr, _ptr]),
    "rexsim_get_state": (C.c_int, [_ptr] * 4),
    "rexsim_set_state": (C.c_int, [_ptr] * 3),
    "rexsim_state_buffers": (C.c_int, [_ptr, _out(_ptr), _out(_ptr)]),
    "rexsim_error_flags": (C.c_int, [_ptr, _out(_ptr)]),
    "rexsim_clear_errors": (C.c_int, [_ptr, _ptr]),
    "rexsim_last_command": (C.c_int, [_ptr, _out(_ptr)]),
    "rexsim_solver_cost": (C.c_int, [_ptr, _out(_ptr)]),
    "rexsim_value_row": (C.c_int, [C.c_char_p]),
    "rexsim_set_env_values": (C.c_int, [_ptr] * 4),
    "rexsim_set_task_values": (C.c_int, [_ptr, _ptr, _i32, _ptr, _u32, _ptr]),
    "rexsim_env_value_buffers": (C.c_int, [_ptr, _out(_ptr), _out(_ptr), _out(_ptr), _out(_i32)]),
    "rexsim_set_env_latencies": (C.c_int, [_ptr] * 3),
    "rexsim_env_latency_buffers": (C.c_int, [_ptr, _out(_ptr), _out(_i32)]),
    "rexsim_set_env_terrains": (C.c_int, [_ptr, _ptr, _f32]),
    "rexsim_env_terrain_buffers": (C.c_int, [_ptr, _out(_ptr), _out(_i32)]),
    "rexsim_set_env_repeats": (C.c_int, [_ptr] * 3),
    "rexsim_env_repeat_buffers": (C.c_int, [_ptr, _out(_ptr)]),
    "rexsim_set_env_tasks": (C.c_int, [_ptr] * 3),
    "rexsim_env_task_buffers": (C.c_int, [_ptr, _out(_ptr)]),
    "rexsim_launch_group_task": (C.c_int, [_ptr, _i32, _out(_i32), _out(_i32)]),
    "rexsim_set_env_marks": (C.c_int, [_ptr] * 2),
    "rexsim_env_mark_buffers": (C.c_int, [_ptr, _out(_ptr)]),
    "rexsim_launch_group_mark": (C.c_int, [_ptr, _i32, _out(_i32)]),
    "rexsim_launch_groups": (C.c_int, [_ptr]),
    "rexsim_launch_group": (C.c_int, [_ptr, _i32, _ptr]),
    "rexsim_slot_buffers": (C.c_int, [_ptr, _out(_ptr), _out(_ptr)]),
    "rexsim_launch_count": (_i64, [_ptr]),
    "rexsim_last_step_build": (C.c_int, [_ptr] + [_out(_i32)] * 3),
    "rexsim_last_terrain_build": (C.c_int, [_ptr, _i32] + [_out(_i32)] * 3),
    "rexsim_last_error": (C.c_char_p, []),
    "rexsim_rand_u32": (_u32, [_u64, _u32, _u32, _u32]),
    "rexsim_noise": (_f32, [_u64] + [_u32] * 5),
    "rexsim_history_depth": (C.c_int, [_sim_cfg]),
    "rexsim_history_buffer": (C.c_int, [_ptr, _out(_ptr), _out(_i64)]),
    "rexsim_set_render_tables": (C.c_int, [_ptr, _ptr, _i32]),
    "rexsim_render": (C.c_int, [_ptr, _ptr, _i32, _i32, _i32, _f32, _f32, _f32, _ptr, _ptr]),
    "rexsim_episode_buffers": (C.c_int, [_ptr] + [_out(_ptr)] * 5 + [_out(_i64)]),
    "rexsim_episode_summary": (C.c_int, [_ptr, _i32, _ptr]),
    "rexsim_set_frames": (C.c_int, [_ptr, _ptr, _i32, _i32]),
    "rexsim_out_dim": (C.c_int, [_ptr]),
    "rexsim_frame_buffers": (C.c_int, [_ptr, _out(_ptr), _out(_i64), _out(_ptr), _out(_i64)]),
    "rexagent_policy_floats": (_i64, [_agent_cfg]),
    "rexagent_value_floats": (_i64, [_agent_cfg]),
    "rexagent_create": (C.c_int, [_agent_cfg, _out(_ptr)]),
    "rexagent_destroy": (None, [_ptr]),
    "rexagent_set_precision": (C.c_int, [_ptr, _i32]),
    "rexagent_set_params": (C.c_int, [_ptr, _ptr, _i64]),
    "rexagent_get_params": (C.c_int, [_ptr, _ptr, _i64]),
    "rexagent_params_buffer": (C.c_int, [_ptr, _out(_ptr)]),
    "rexagent_state_buffers": (C.c_int, [_ptr, _out(_ptr), _out(_ptr)]),
    "rexagent_set_filters": (C.c_int, [_ptr, _i64, _ptr, _ptr, _i64, _f32, _f32]),
    "rexagent_get_filters": (C.c_int, [_ptr] * 5),
    "rexagent_perform": (C.c_int, [_ptr, _ptr, _i32, _i32, _u64, _u32, _u32] + [_ptr] * 6),
    "rexagent_experience": (C.c_int, [_ptr, _ptr, _ptr, _i32, _ptr]),
    "rexagent_experience_partial": (C.c_int, [_ptr, _ptr, _ptr, _i32, _ptr, _ptr]),
    "rexagent_experience_finalize": (C.c_int, [_ptr, _ptr, _i32, _ptr, _ptr, _ptr]),
    "rexagent_transform_reward": (C.c_int, [_ptr, _ptr, _i32, _ptr, _ptr]),
    "rexagent_discounted_return": (C.c_int, [_ptr, _ptr, _i32, _i32, _i64, _i64, _f32, _ptr, _ptr]),
    "rexagent_lambda_advantage": (C.c_int, [_ptr, _ptr, _ptr, _i32, _i32, _i64, _i64, _f32, _ptr, _ptr]),
    "rexagent_gae_segments": (C.c_int, [_ptr, _ptr, _ptr, _i32, _i32, _f32, _f32, _ptr, _ptr, _ptr]),
    "rexsim_gae_segments_bootstrap": (C.c_int, [_ptr] * 5 + [_i32, _i32, _f32, _f32, _ptr, _ptr, _ptr]),
    "rexagent_launch_count": (_i64, [_ptr]),
    "rexrnn_policy_floats": (_i64, [_agent_cfg, _rnn_cfg]),
    "rexrnn_check": (C.c_int, [_agent_cfg, _rnn_cfg]),
    "rexrnn_create": (C.c_int, [_ptr, _rnn_cfg, _out(_ptr)]),
    "rexrnn_destroy": (None, [_ptr]),
    "rexrnn_set_params": (C.c_int, [_ptr, _ptr, _i64]),
    "rexrnn_get_params": (C.c_int, [_ptr, _ptr, _i64]),
    "rexrnn_state_buffer": (C.c_int, [_ptr, _out(_ptr)]),
    "rexrnn_perform": (C.c_int, [_ptr, _ptr, _ptr, _i32, _i32, _u64, _u32, _u32] + [_ptr] * 6),
    "rexrnn_launch_count": (_i64, [_ptr]),
}
EXPORTS = [n for n in SIGNATURES if n.startswith("rexsim_")]
AGENT_EXPORTS = [n for n in SIGNATURES if n.startswith("rexagent_")]
RNN_EXPORTS = [n for n in SIGNATURES if n.startswith("rexrnn_")]

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
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    _LIB = L
    return L


def check(rc):
    if rc == 0:
        return
    msg = load().rexsim_last_error().decode()
    if rc in (-1, -2, -4):
        raise ValueError(f"rexsim: {msg} (status {rc})")
    raise RuntimeError(f"rexsim: {msg} (status {rc})")


class DevArray(object):
    """Expose a raw device pointer to torch through __cuda_array_interface__ (no copy, no ownership)."""

    def __init__(self, ptr, shape, typestr, owner):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 2}
        self._owner = owner


def device_view(ptr, shape, typestr, owner, device):
    """torch tensor over raw device memory of a handle; the view keeps `owner` alive."""
    return torch.as_tensor(DevArray(ptr, shape, typestr, owner), device=device)


def stream_ptr(device):
    """The current torch stream of `device`, as the `void* stream` argument of the C ABI."""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def call(index, fn, *args, stream=True):
    """fn(*args[, current stream]) with CUDA device `index` current, raising on a non-zero status.  The device is only
    entered when it is not the current one already, which is what a step costs least."""
    if torch.cuda.current_device() == index:
        rc = fn(*args, torch.cuda.current_stream().cuda_stream) if stream else fn(*args)
    else:
        with torch.cuda.device(index):
            rc = fn(*args, torch.cuda.current_stream().cuda_stream) if stream else fn(*args)
    if rc:
        check(rc)
