"""ctypes binding of librlca.so (the C ABI declared in include/rlca.h).

PyTorch is plumbing here: it owns device memory and streams; the library gets
raw pointers.  There is NO fallback: if the shared library is missing or a
call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'librlca.so')


class RlcaError(RuntimeError):
    pass


class EnvConfig(C.Structure):
    """Mirror of rlca_env_config (include/rlca.h)."""
    _fields_ = [
        ('robots_per_world', C.c_int32), ('num_worlds', C.c_int32),
        ('beams', C.c_int32), ('raw_beams', C.c_int32),
        ('grid_w', C.c_int32), ('grid_h', C.c_int32),
        ('origin_cx', C.c_int32), ('origin_cy', C.c_int32),
        ('resolution', C.c_float), ('ppm', C.c_float),
        ('dt', C.c_float), ('inv_dt', C.c_float),
        ('range_max', C.c_float), ('range_cells', C.c_float),
        ('fov', C.c_float),
        ('half_len', C.c_float), ('half_wid', C.c_float),
        ('goal_radius', C.c_float), ('reward_arrive', C.c_float),
        ('reward_collision', C.c_float), ('progress_gain', C.c_float),
        ('w_threshold', C.c_float), ('w_penalty', C.c_float),
        ('v_min', C.c_float), ('v_max', C.c_float), ('w_min', C.c_float), ('w_max', C.c_float),
        ('timeout', C.c_int32), ('pre_distance_zero', C.c_int32),
        ('scenario', C.c_int32), ('auto_reset', C.c_int32),
        ('max_reject', C.c_int32), ('world_offset', C.c_int32),
        ('seed', C.c_uint64),
    ]


class EnvState(C.Structure):
    _fields_ = [('pose_dev', C.c_void_p), ('goal_dev', C.c_void_p),
                ('acc_dev', C.c_void_p), ('meta_dev', C.c_void_p)]


class StepIO(C.Structure):
    _fields_ = [('action_dev', C.c_void_p), ('live_dev', C.c_void_p), ('obs_dev', C.c_void_p),
                ('reward_dev', C.c_void_p), ('flags_dev', C.c_void_p), ('gs_dev', C.c_void_p),
                ('eplog_dev', C.c_void_p), ('stack_in_dev', C.c_void_p), ('stack_out_dev', C.c_void_p)]


class EvalState(C.Structure):
    """Mirror of rlca_eval_state (include/rlca.h)."""
    _fields_ = [('path_dev', C.c_void_p), ('count_dev', C.c_void_p), ('closed_dev', C.c_void_p),
                ('open_dev', C.c_void_p), ('records_dev', C.c_void_p), ('episodes', C.c_int32)]


class DemoSet(C.Structure):
    """Mirror of rlca_demo_set (include/rlca.h)."""
    _fields_ = [('obs_dev', C.c_void_p), ('gs_dev', C.c_void_p), ('action_dev', C.c_void_p),
                ('count_dev', C.c_void_p), ('capacity', C.c_int64)]


class LayoutParams(C.Structure):
    """Mirror of rlca_layout_params (include/rlca.h)."""
    _fields_ = [('side', C.c_float), ('separation', C.c_float), ('min_travel', C.c_float)]


class ArenaTables(C.Structure):
    """Mirror of rlca_arena_tables (include/rlca.h)."""
    _fields_ = [('num_arenas', C.c_int32), ('cell_off', C.c_void_p), ('cells', C.c_void_p)]


class HybridParams(C.Structure):
    """Mirror of rlca_hybrid_params (include/rlca.h)."""
    _fields_ = [('r_safe', C.c_float), ('r_risk', C.c_float), ('v_safe', C.c_float), ('heading_gain', C.c_float)]


class SafetyParams(C.Structure):
    """Mirror of rlca_safety_params (include/rlca.h)."""
    _fields_ = [('near_dist', C.c_float)]


class SafetyState(C.Structure):
    """Mirror of rlca_safety_state (include/rlca.h)."""
    _fields_ = [('min_sep_dev', C.c_void_p), ('min_clear_dev', C.c_void_p), ('last_clear_dev', C.c_void_p),
                ('near_dev', C.c_void_p), ('partner_dev', C.c_void_p), ('records_dev', C.c_void_p),
                ('episodes', C.c_int32)]


class ProgressParams(C.Structure):
    """Mirror of rlca_progress_params (include/rlca.h)."""
    _fields_ = [('window', C.c_int32), ('progress_dist', C.c_float), ('still_dist', C.c_float),
                ('block_dist', C.c_float)]


class ProgressState(C.Structure):
    """Mirror of rlca_progress_state (include/rlca.h)."""
    _fields_ = [('running_dev', C.c_void_p), ('counters_dev', C.c_void_p), ('records_dev', C.c_void_p),
                ('causes_dev', C.c_void_p), ('episodes', C.c_int32)]


class NoiseParams(C.Structure):
    """Mirror of rlca_noise_params (include/rlca.h)."""
    _fields_ = [('range_sigma', C.c_float), ('dropout', C.c_float), ('v_gain_sigma', C.c_float),
                ('w_gain_sigma', C.c_float), ('seed', C.c_uint64), ('stream_id', C.c_uint32)]


class LatencyParams(C.Structure):
    """Mirror of rlca_latency_params (include/rlca.h)."""
    _fields_ = [('scan_lo', C.c_int32), ('scan_hi', C.c_int32), ('cmd_lo', C.c_int32), ('cmd_hi', C.c_int32),
                ('seed', C.c_uint64), ('stream_id', C.c_uint32)]


class LatencyState(C.Structure):
    """Mirror of rlca_latency_state (include/rlca.h): device pointers, or host pointers for the host twins."""
    _fields_ = [('scan_ring', C.c_void_p), ('cmd_ring', C.c_void_p), ('scan_delay', C.c_void_p),
                ('cmd_delay', C.c_void_p)]


class DynamicsParams(C.Structure):
    """Mirror of rlca_dynamics_params (include/rlca.h)."""
    _fields_ = [('lin_lo', C.c_float), ('lin_hi', C.c_float), ('ang_lo', C.c_float), ('ang_hi', C.c_float),
                ('seed', C.c_uint64), ('stream_id', C.c_uint32)]


class DynamicsState(C.Structure):
    """Mirror of rlca_dynamics_state (include/rlca.h): device pointers, or host pointers for the host twin."""
    _fields_ = [('vel', C.c_void_p), ('lin_limit', C.c_void_p), ('ang_limit', C.c_void_p)]


class CrowdParams(C.Structure):
    """Mirror of rlca_crowd_params (include/rlca.h)."""
    _fields_ = [(k, C.c_float) for k in ('speed', 'relax_time', 'strength', 'range', 'anisotropy', 'side_bias', 'radius',
                                         'neighbour_dist', 'wall_strength', 'wall_range', 'wall_dist', 'heading_gain')] + \
        [('see_robots', C.c_int32)]


class LocalizationParams(C.Structure):
    """Mirror of rlca_localization_params (include/rlca.h)."""
    _fields_ = [('xy_lo', C.c_float), ('xy_hi', C.c_float), ('theta_lo', C.c_float), ('theta_hi', C.c_float),
                ('tau', C.c_float), ('v_sigma', C.c_float), ('w_sigma', C.c_float), ('seed', C.c_uint64),
                ('stream_id', C.c_uint32)]


class DwaParams(C.Structure):
    """Mirror of rlca_dwa_params (include/rlca.h)."""
    _fields_ = [('v_samples', C.c_int32), ('w_samples', C.c_int32)] + \
        [(k, C.c_float) for k in ('radius', 'horizon', 'heading_time', 'accel', 'angular_accel', 'brake',
                                  'heading_weight', 'clearance_weight', 'speed_weight', 'clearance_cap')]


class PlanTables(C.Structure):
    """Mirror of rlca_plan_tables (include/rlca.h)."""
    _fields_ = [('num_components', C.c_int32), ('max_area', C.c_int32), ('label', C.c_void_p), ('rects', C.c_void_p)]


class PlanState(C.Structure):
    """Mirror of rlca_plan_state (include/rlca.h): device pointers, or host pointers for the host twins."""
    _fields_ = [('entry', C.c_void_p), ('rect', C.c_void_p), ('field', C.c_void_p), ('list', C.c_void_p),
                ('status', C.c_void_p), ('status_count', C.c_void_p), ('length', C.c_void_p), ('records', C.c_void_p),
                ('episodes', C.c_int32)]


class LocalizationState(C.Structure):
    """Mirror of rlca_localization_state (include/rlca.h): device pointers, or host pointers for the host twin."""
    _fields_ = [('err', C.c_void_p), ('sigma', C.c_void_p)]


# rlca_eval_reduce partials per world (the RLCA_EVAL_* columns of include/rlca.h)
EVAL_PARTIALS = ('reached', 'crashed', 'timed_out', 'unfinished', 'sum_time', 'sum_time_sq', 'sum_extra_time',
                 'sum_extra_time_sq', 'sum_extra_distance', 'sum_extra_distance_sq', 'sum_speed', 'sum_speed_sq',
                 'sum_straight', 'sum_path')

# rlca_safety_reduce partials per world (the RLCA_SAFETY_* columns of include/rlca.h); the last one is a minimum
SAFETY_PARTIALS = ('crash_static', 'crash_robot', 'crash_both_in_range', 'crash_into_masked', 'reached',
                   'reached_separation', 'sum_separation', 'sum_separation_sq', 'reached_clearance', 'sum_clearance',
                   'sum_clearance_sq', 'near_episodes', 'sum_near_ticks', 'min_separation')

# rlca_progress_reduce partials per world (the RLCA_PROGRESS_* columns of include/rlca.h), all sums
PROGRESS_PARTIALS = tuple(g + '_' + k for g in ('timeout', 'unfinished')
                          for k in ('frozen', 'stalled', 'slow', 'robot_near', 'folded', 'sum_closest',
                                    'sum_closest_sq')) + \
    ('sum_still_ticks', 'sum_ticks', 'reached', 'sum_rotation', 'sum_rotation_sq')

# rlca_plan_reduce partials per world (the RLCA_PLAN_* columns of include/rlca.h), all sums
PLAN_PARTIALS = ('reached', 'sum_length', 'sum_extra', 'sum_extra_sq', 'no_path')

# every symbol include/rlca.h declares: (name, restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    'rlca_walk_tables_host': (C.c_int, [C.c_float, _P, _P, _P, _P, _P, _P, _P]),
    'rlca_inv_records_host': (C.c_int, [C.c_float, _P, _P, _P, _P]),
    'rlca_env_create': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(_P)]),
    'rlca_env_destroy': (C.c_int, [_P]),
    'rlca_env_set_map': (C.c_int, [_P, _P, C.c_int32, C.c_int32]),
    'rlca_env_set_tables': (C.c_int, [_P, _P, _P]),
    'rlca_env_reset': (C.c_int, [_P, C.POINTER(EnvState), _P, C.c_int32, _P]),
    'rlca_env_observe': (C.c_int, [_P, C.POINTER(EnvState), C.POINTER(StepIO), _P]),
    'rlca_env_step': (C.c_int, [_P, C.POINTER(EnvState), C.POINTER(EnvState), C.POINTER(StepIO), _P]),
    'rlca_env_step_host': (C.c_int, [_P, C.POINTER(EnvState), C.POINTER(EnvState), C.POINTER(StepIO),
                                     _P, _P, _P, _P, _P, _P]),
    'rlca_raycast': (C.c_int, [_P, _P, _P, C.c_int32, _P]),
    'rlca_env_set_ctas_per_world': (C.c_int, [_P, C.c_int32]),
    'rlca_env_set_host_chunks': (C.c_int, [_P, C.c_int32]),
    'rlca_env_set_host_zero_copy': (C.c_int, [_P, C.c_int32]),
    'rlca_env_launch_count': (C.c_int64, [_P]),
    'rlca_env_lidar_ctas_per_sm': (C.c_int, [_P, C.POINTER(C.c_int32)]),
    'rlca_sizeof_env_config': (C.c_int, []),
    'rlca_policy_param_offset': (C.c_int64, [C.c_int32]),
    'rlca_policy_param_size': (C.c_int64, [C.c_int32]),
    'rlca_policy_launch_count': (C.c_int64, [_P]),
    'rlca_policy_set_grad_event': (C.c_int, [_P, _P]),
    'rlca_adam_step_allreduce': (C.c_int, [_P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int32, C.c_int32,
                                           C.c_int64, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int32, C.c_float, C.c_int32, _P]),
    'rlca_policy_set_tensor_cores': (C.c_int, [_P, C.c_int32]),
    'rlca_policy_weights_changed': (C.c_int, [_P]),
    'rlca_policy_features': (C.c_int, [_P, C.c_int32, C.c_int32, _P, _P]),
    'rlca_policy_create': (C.c_int, [C.c_int32, C.POINTER(_P)]),
    'rlca_policy_destroy': (C.c_int, [_P]),
    'rlca_policy_forward': (C.c_int, [_P, _P, _P, _P, C.c_int32, _P, _P, _P]),
    'rlca_policy_sample': (C.c_int, [_P, _P, C.c_int32, C.c_uint64, C.c_uint64, C.c_int32, _P, _P, _P, _P]),
    'rlca_ppo_loss_fwd_bwd': (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, C.c_int32, C.c_float, C.c_float, C.c_float,
                                        _P, _P]),
    'rlca_ppo_loss_fwd_bwd_weighted': (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, C.c_int32, C.c_float, C.c_float,
                                                 C.c_float, C.c_float, _P, _P]),
    'rlca_ppo_diag_accumulate': (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, C.c_int32, C.c_float, _P, _P, _P]),
    'rlca_grad_sumsq': (C.c_int, [_P, _P, _P, _P]),
    'rlca_bc_loss_fwd_bwd': (C.c_int, [_P, _P, _P, _P, C.c_int32, _P, _P]),
    'rlca_policy_backward': (C.c_int, [_P, _P, _P, _P, C.c_int32, _P, _P]),
    'rlca_adam_step': (C.c_int, [_P, _P, _P, _P, C.c_int64, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int32,
                                 C.c_float, _P]),
    'rlca_policy_adam_step': (C.c_int, [_P, _P, _P, _P, _P, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int32,
                                        C.c_float, _P]),
    'rlca_gae': (C.c_int, [_P, _P, _P, _P, C.c_int32, C.c_int32, C.c_float, C.c_float, _P, _P, _P]),
    'rlca_adv_moments': (C.c_int, [_P, C.c_int64, _P, _P]),
    'rlca_adv_apply': (C.c_int, [_P, C.c_int64, _P, _P, _P]),
    'rlca_gather_rows': (C.c_int, [_P, _P, C.c_int32, C.c_int32, _P, _P]),
    'rlca_gather_minibatch': (C.c_int, [_P, _P, C.c_int32, _P, C.c_int32, _P, _P]),
    'rlca_obs_stack_push': (C.c_int, [_P, _P, _P, C.c_int32, C.c_int32, _P, _P]),
    'rlca_eval_track': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(EnvState), C.POINTER(EnvState), C.POINTER(StepIO),
                                  C.POINTER(EvalState), _P]),
    'rlca_eval_reduce': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(EvalState), C.c_int32, C.c_int32, _P, _P]),
    'rlca_eval_reduce_host': (C.c_int, [C.POINTER(EnvConfig), _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    'rlca_eval_reduce_split': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(EvalState), _P, C.c_int32, C.c_int32, _P,
                                         _P]),
    'rlca_eval_reduce_split_host': (C.c_int, [C.POINTER(EnvConfig), _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32,
                                              _P]),
    'rlca_orca_action': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(EnvState), C.c_float, C.c_float, C.c_float,
                                   C.c_float, _P, _P, _P, _P]),
    'rlca_orca_action_host': (C.c_int, [C.POINTER(EnvConfig), _P, _P, _P, C.c_float, C.c_float, C.c_float, C.c_float,
                                        _P, _P, _P]),
    'rlca_noncoop_action': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(EnvState), _P, C.c_float, C.c_float, _P, _P]),
    'rlca_noncoop_action_host': (C.c_int, [C.POINTER(EnvConfig), _P, _P, _P, _P, C.c_float, C.c_float, _P]),
    'rlca_crowd_action': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(CrowdParams), C.POINTER(EnvState), _P, _P, _P,
                                    _P]),
    'rlca_crowd_action_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(CrowdParams), _P, _P, _P, _P, _P, _P]),
    'rlca_crowd_expf_host': (C.c_int, [_P, C.c_int32, _P]),
    'rlca_hybrid_action': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(HybridParams), C.POINTER(EnvState), _P, _P, _P,
                                     _P, _P, _P]),
    'rlca_hybrid_action_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(HybridParams), _P, _P, _P, _P, _P, _P, _P,
                                          _P]),
    'rlca_nh_orca_action': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(EnvState), C.c_float, C.c_float, C.c_float,
                                      C.c_float, C.c_float, _P, _P, _P, _P]),
    'rlca_nh_orca_action_host': (C.c_int, [C.POINTER(EnvConfig), _P, _P, _P, C.c_float, C.c_float, C.c_float,
                                           C.c_float, C.c_float, _P, _P, _P]),
    'rlca_nh_orca_polygon_host': (C.c_int, [C.POINTER(EnvConfig), C.c_float, C.c_float, _P, _P]),
    'rlca_orca_obstacles_create': (C.c_int, [C.POINTER(EnvConfig), _P, C.c_int32, C.c_int32, C.c_float,
                                             C.POINTER(_P)]),
    'rlca_orca_obstacles_destroy': (C.c_int, [_P]),
    'rlca_orca_obstacles_segments': (C.c_int, [_P, _P, _P, _P, _P]),
    'rlca_orca_action_map': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(EnvState), _P, C.c_float, C.c_float,
                                       C.c_float, C.c_float, C.c_float, _P, _P, _P, _P]),
    'rlca_orca_action_map_host': (C.c_int, [C.POINTER(EnvConfig), _P, _P, _P, _P, C.c_float, C.c_float, C.c_float,
                                            C.c_float, C.c_float, _P, _P, _P]),
    'rlca_nh_orca_action_map': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(EnvState), _P, C.c_float, C.c_float,
                                          C.c_float, C.c_float, C.c_float, C.c_float, _P, _P, _P, _P]),
    'rlca_nh_orca_action_map_host': (C.c_int, [C.POINTER(EnvConfig), _P, _P, _P, _P, C.c_float, C.c_float,
                                               C.c_float, C.c_float, C.c_float, C.c_float, _P, _P, _P]),
    'rlca_orca_obstacle_lines_host': (C.c_int, [C.POINTER(EnvConfig), _P, _P, _P, _P, C.c_int32, C.c_float,
                                                C.c_float, _P, _P, _P]),
    'rlca_demo_append': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(EnvState), C.POINTER(StepIO), C.POINTER(DemoSet),
                                   _P]),
    'rlca_layout_random': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LayoutParams), C.POINTER(EnvState), _P, _P]),
    'rlca_layout_random_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LayoutParams), _P, _P, _P, _P]),
    'rlca_layout_respawn': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LayoutParams), C.POINTER(EnvState), _P, _P, _P,
                                      _P]),
    'rlca_layout_respawn_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LayoutParams), _P, _P, _P, _P, _P, _P,
                                           _P]),
    'rlca_stack_refresh': (C.c_int, [C.POINTER(EnvConfig), _P, _P, _P, _P, _P, _P]),
    'rlca_arena_tables_check': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(ArenaTables)]),
    'rlca_layout_arena': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LayoutParams), C.POINTER(ArenaTables), C.c_int32,
                                    C.POINTER(EnvState), _P, _P]),
    'rlca_layout_arena_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LayoutParams), C.POINTER(ArenaTables),
                                         C.c_int32, _P, _P, _P, _P]),
    'rlca_layout_arena_respawn': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LayoutParams), C.POINTER(ArenaTables),
                                            C.c_int32, C.POINTER(EnvState), _P, _P, _P, _P]),
    'rlca_layout_arena_respawn_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LayoutParams),
                                                 C.POINTER(ArenaTables), C.c_int32, _P, _P, _P, _P, _P, _P, _P]),
    'rlca_safety_track': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(SafetyParams), C.POINTER(EnvState),
                                    C.POINTER(EnvState), C.POINTER(StepIO), C.POINTER(EvalState),
                                    C.POINTER(SafetyState), _P]),
    'rlca_safety_track_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(SafetyParams), _P, _P, _P, _P, _P, _P, _P,
                                         C.c_int32, _P, _P, _P, _P, _P, _P]),
    'rlca_safety_separation_host': (C.c_int, [C.POINTER(EnvConfig), _P, _P, C.c_int32, _P]),
    'rlca_safety_contact_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(C.c_float)]),
    'rlca_safety_reduce': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(SafetyState), C.POINTER(EvalState), _P, C.c_int32,
                                     C.c_int32, _P, _P]),
    'rlca_safety_reduce_host': (C.c_int, [C.POINTER(EnvConfig), _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    'rlca_progress_track': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(ProgressParams), C.POINTER(EnvState),
                                      C.POINTER(EnvState), C.POINTER(StepIO), C.POINTER(EvalState),
                                      C.POINTER(ProgressState), _P]),
    'rlca_progress_track_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(ProgressParams), _P, _P, _P, _P, _P, _P,
                                           C.c_int32, _P, _P, _P, _P]),
    'rlca_progress_reduce': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(ProgressParams), C.POINTER(ProgressState),
                                       C.POINTER(EvalState), _P, C.c_int32, C.c_int32, _P, _P]),
    'rlca_progress_reduce_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(ProgressParams), _P, _P, _P, _P, _P, _P,
                                            _P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    'rlca_noise_scan': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(NoiseParams), C.c_uint32, _P, _P, _P]),
    'rlca_noise_action': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(NoiseParams), C.c_uint32, _P, _P, _P]),
    'rlca_noise_scan_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(NoiseParams), C.c_uint32, _P, _P]),
    'rlca_noise_action_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(NoiseParams), C.c_uint32, _P, _P]),
    'rlca_latency_scan': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LatencyParams), C.POINTER(LatencyState),
                                    C.c_uint32, _P, _P, _P]),
    'rlca_latency_action': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LatencyParams), C.POINTER(LatencyState),
                                      C.c_uint32, _P, _P, _P, _P]),
    'rlca_latency_scan_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LatencyParams), C.POINTER(LatencyState),
                                         C.c_uint32, _P, _P]),
    'rlca_latency_action_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LatencyParams), C.POINTER(LatencyState),
                                           C.c_uint32, _P, _P, _P]),
    'rlca_dynamics_action': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(DynamicsParams), C.POINTER(DynamicsState),
                                       C.c_uint32, _P, _P, _P, _P]),
    'rlca_dynamics_action_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(DynamicsParams),
                                            C.POINTER(DynamicsState), C.c_uint32, _P, _P, _P]),
    'rlca_localization_observe': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LocalizationParams),
                                            C.POINTER(LocalizationState), C.c_uint32, _P, C.POINTER(EnvState), _P,
                                            _P, _P]),
    'rlca_localization_observe_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(LocalizationParams),
                                                 C.POINTER(LocalizationState), C.c_uint32, _P, C.POINTER(EnvState),
                                                 _P, _P]),
    'rlca_dwa_action': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(DwaParams), _P, _P, _P, _P, _P, _P]),
    'rlca_dwa_action_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(DwaParams), _P, _P, _P, _P, _P, _P, _P]),
    'rlca_plan_tables_check': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(PlanTables)]),
    'rlca_plan_fields': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(PlanTables), C.POINTER(PlanState),
                                   C.POINTER(EnvState), _P]),
    'rlca_plan_fields_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(PlanTables), C.POINTER(PlanState),
                                        C.POINTER(EnvState)]),
    'rlca_plan_waypoints': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(PlanTables), C.POINTER(PlanState),
                                      C.POINTER(EnvState), _P, _P, _P]),
    'rlca_plan_waypoints_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(PlanTables), C.POINTER(PlanState),
                                           C.POINTER(EnvState), _P, _P]),
    'rlca_plan_shape': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(PlanTables), C.POINTER(PlanState), _P, _P,
                                  C.POINTER(EnvState), _P, _P, _P, _P, _P, _P]),
    'rlca_plan_shape_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(PlanTables), C.POINTER(PlanState), _P, _P,
                                       C.POINTER(EnvState), _P, _P, _P, _P, _P]),
    'rlca_plan_track': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(PlanTables), C.POINTER(PlanState),
                                  C.POINTER(EnvState), C.POINTER(EnvState), _P, C.POINTER(EvalState), _P]),
    'rlca_plan_track_host': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(PlanTables), C.POINTER(PlanState),
                                       C.POINTER(EnvState), C.POINTER(EnvState), _P, _P, _P, C.c_int32]),
    'rlca_plan_reduce': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(PlanState), C.POINTER(EvalState), C.c_int32,
                                   C.c_int32, _P, _P]),
    'rlca_plan_reduce_split': (C.c_int, [C.POINTER(EnvConfig), C.POINTER(PlanState), C.POINTER(EvalState), _P,
                                         C.c_int32, C.c_int32, _P, _P]),
    'rlca_plan_reduce_host': (C.c_int, [C.POINTER(EnvConfig), _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P]),
    'rlca_last_error': (C.c_char_p, []),
    'rlca_version': (C.c_char_p, []),
}

_lib = None


def load():
    """Load librlca.so (built in-tree by __graft_entry__.build()). Raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RlcaError(f'{LIB_PATH} not found: run `python -c "import __graft_entry__ as g; g.build()"` '
                        '(there is no CPU fallback)')
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)      # AttributeError if the export is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int):
    if rc != 0:
        msg = load().rlca_last_error()
        raise RlcaError(f'librlca error {rc}: {msg.decode() if msg else "?"}')
