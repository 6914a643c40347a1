"""ctypes binding of libfenerf_b200.so (include/fenerf_b200.h).

The library is a plain C-ABI shared object built in-tree by ``fenerf_b200.build``; this module
declares its structs and prototypes and fails loudly when the library is missing -- there is no
CPU or PyTorch fallback on the render path.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FENERF_B200_LIB") or os.path.join(_HERE, "libfenerf_b200.so")   # env: experiment builds only

MAX_TRUNK, MAX_COLOR, MAX_LABEL, HIDDEN = 8, 8, 32, 256

ABI_VERSION = 3
FIELD_LABEL_FILM = 0x1        # fenerf_field_desc.reserved (the flags word): FENERF_FIELD_LABEL_FILM
FIELD_GRID_TRUNK = 0x2        # FENERF_FIELD_GRID_TRUNK: the grid features feed the first trunk layer
FIELD_BRIDGE = 0x4            # FENERF_FIELD_BRIDGE: the colour branch starts from v = Linear(256 -> 3)(trunk output)
FIELD_FEATURE_HEAD = 0x8      # FENERF_FIELD_FEATURE_HEAD: Linear(256 -> 64) colour head without the sigmoid
FIELD_BRIDGE_RES = 0x10       # FENERF_FIELD_BRIDGE_RES: v adds the position, the density is a Linear chain on v
FIELD_WO_DIR = 0x20           # FENERF_FIELD_WO_DIR: the first colour layer reads [feat, x], no ray direction
FIELD_SPLIT_IMAGES = 0x40     # FENERF_FIELD_SPLIT_IMAGES: the pack also holds the fp16 low parts of the weight images
PRECISION = {"exact": 0, "fast": 1, "guard": 2, "split": 3}
CLAMP = {"relu": 0, "softplus": 1}
FILL_MODE = {None: 0, "debug": 1, "weight": 2, "weight_debug": 3, "seg_padding_background": 4,
             "eval_seg_padding_background": 5, "eval_white_back": 6}
FILL_COLOR = {"black": 0.0, "white": 1.0, "grey": 0.5, "light_grey": 0.81}
E_CLAMP_MODE = -5
CAMERA_MODE = {"uniform": 1, "normal": 2, "gaussian": 2, "truncated_gaussian": 3, "spherical_uniform": 4}

EXPORTS = (
    "fenerf_packed_bytes", "fenerf_pack_field", "fenerf_siren_points", "fenerf_ray_setup", "fenerf_resample",
    "fenerf_composite", "fenerf_workspace_bytes", "fenerf_render_forward", "fenerf_last_error",
    "fenerf_abi_version", "fenerf_launch_count", "fenerf_camera_poses",
    "fenerf_field_fingerprint", "fenerf_composite_backward", "fenerf_film_forward_stash", "fenerf_gate_backward",
    "fenerf_head_grads", "fenerf_extras_gather", "fenerf_grid_scatter_add", "fenerf_grid_unpack_grad",
    "fenerf_workspace_layout", "fenerf_mask2color", "fenerf_frames_to_u8", "fenerf_mapping_film",
    "fenerf_guard_stats", "fenerf_debug_stage_times", "fenerf_debug_fast_variant", "fenerf_debug_soft_sine",
    "fenerf_gemm_nt_f16", "fenerf_gemm_nt_film", "fenerf_gemm_tn_f16",
    "fenerf_gemm_nt_split", "fenerf_gemm_nt_film_split", "fenerf_gemm_tn_split", "fenerf_absmax_f32",
    "fenerf_pack_field_bridge", "fenerf_field_fingerprint_bridge",
    "fenerf_render_rays", "fenerf_rays_workspace_bytes", "fenerf_rays_workspace_layout", "fenerf_composite_backward_rays",
    "fenerf_gate_backward_det", "fenerf_absmax_finite", "fenerf_grid_scatter_det_workspace_bytes",
    "fenerf_grid_scatter_add_det", "fenerf_det_launch_count",
    "fenerf_render_rays_grad", "fenerf_rays_grad_workspace_layout", "fenerf_composite_backward_rays_dz",
    "fenerf_grid_coord_grad", "fenerf_ray_dir_grad",
    "fenerf_mc_workspace_bytes", "fenerf_mc_count", "fenerf_mc_emit",
)


class FieldDesc(C.Structure):
    _fields_ = [("trunk_layers", C.c_int32), ("color_layers", C.c_int32), ("label_dim", C.c_int32),
                ("grid_channels", C.c_int32), ("grid_res", C.c_int32), ("out_dim", C.c_int32),
                ("input_scale", C.c_float), ("reserved", C.c_int32)]


class FieldParams(C.Structure):
    _fields_ = [("trunk_w", C.c_void_p * MAX_TRUNK), ("trunk_b", C.c_void_p * MAX_TRUNK),
                ("sigma_w", C.c_void_p), ("sigma_b", C.c_void_p),
                ("color_w", C.c_void_p * MAX_COLOR), ("color_b", C.c_void_p * MAX_COLOR),
                ("rgb_w", C.c_void_p), ("rgb_b", C.c_void_p),
                ("label_w", C.c_void_p * 3), ("label_b", C.c_void_p * 3),
                ("grid", C.c_void_p)]


class BridgeParams(C.Structure):
    _fields_ = [("density_w", C.c_void_p * 4), ("density_b", C.c_void_p * 4), ("pre_w", C.c_void_p), ("pre_b", C.c_void_p)]


class RenderDesc(C.Structure):
    _fields_ = [("batch", C.c_int32), ("img_h", C.c_int32), ("img_w", C.c_int32), ("num_steps", C.c_int32),
                ("hierarchical", C.c_int32), ("clamp_mode", C.c_int32),
                ("last_back", C.c_int32), ("white_back", C.c_int32), ("black_back", C.c_int32),
                ("fill_mode", C.c_int32), ("fill_color", C.c_float), ("softmax_label", C.c_int32),
                ("lock_view_dependence", C.c_int32), ("precision", C.c_int32),
                ("noise_std", C.c_float), ("tan_half_fov", C.c_float), ("guard_tau", C.c_float)]


class GuardReport(C.Structure):
    _fields_ = [("refined", C.c_int32), ("max_abs_delta", C.c_float), ("sign_flips", C.c_int32), ("tau", C.c_float)]


class MappingParams(C.Structure):
    _fields_ = [("weight", C.c_void_p * 5), ("bias", C.c_void_p * 5), ("z_dim", C.c_int32), ("hidden_dim", C.c_int32)]


class WorkspaceOffsets(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("points_coarse", "z_coarse", "dirs", "origins", "raw_coarse", "z_fine",
                                          "points_fine", "raw_fine", "total")]


class RaysWorkspaceOffsets(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("raw_coarse", "z_fine", "points_fine", "dirs_fine", "raw_fine", "total")]


_lib = None


def _declare(lib):
    vp, i32, i64, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t
    P = C.POINTER
    lib.fenerf_packed_bytes.restype = sz
    lib.fenerf_packed_bytes.argtypes = [P(FieldDesc)]
    lib.fenerf_pack_field.restype = C.c_int
    lib.fenerf_pack_field.argtypes = [P(FieldDesc), P(FieldParams), vp, sz, vp]
    lib.fenerf_field_fingerprint.restype = C.c_int
    lib.fenerf_field_fingerprint.argtypes = [P(FieldDesc), P(FieldParams), vp, vp]
    lib.fenerf_pack_field_bridge.restype = C.c_int
    lib.fenerf_pack_field_bridge.argtypes = [P(FieldDesc), P(FieldParams), P(BridgeParams), vp, sz, vp]
    lib.fenerf_field_fingerprint_bridge.restype = C.c_int
    lib.fenerf_field_fingerprint_bridge.argtypes = [P(FieldDesc), P(FieldParams), P(BridgeParams), vp, vp]
    lib.fenerf_siren_points.restype = C.c_int
    lib.fenerf_siren_points.argtypes = [P(FieldDesc), vp, vp, vp, vp, i32, i64, i32, i32, vp, i32, vp, vp]
    lib.fenerf_camera_poses.restype = C.c_int
    lib.fenerf_camera_poses.argtypes = [i32, i32, C.c_float, C.c_float, C.c_float, C.c_float, vp, vp, vp, vp, vp, vp]
    lib.fenerf_ray_setup.restype = C.c_int
    lib.fenerf_ray_setup.argtypes = [P(RenderDesc)] + [vp] * 10
    lib.fenerf_resample.restype = C.c_int
    lib.fenerf_resample.argtypes = [P(RenderDesc), i32] + [vp] * 10
    lib.fenerf_composite.restype = C.c_int
    lib.fenerf_composite.argtypes = [P(RenderDesc), i32] + [vp] * 11
    lib.fenerf_workspace_bytes.restype = sz
    lib.fenerf_workspace_bytes.argtypes = [P(RenderDesc), P(FieldDesc)]
    lib.fenerf_workspace_layout.restype = C.c_int
    lib.fenerf_workspace_layout.argtypes = [P(RenderDesc), P(FieldDesc), P(WorkspaceOffsets)]
    lib.fenerf_render_forward.restype = C.c_int
    lib.fenerf_render_forward.argtypes = [P(RenderDesc), P(FieldDesc)] + [vp] * 15 + [vp, sz, vp]
    lib.fenerf_render_rays.restype = C.c_int
    lib.fenerf_render_rays.argtypes = [P(RenderDesc), P(FieldDesc), vp, vp, vp, vp, i32] + [vp] * 9 + [vp, sz, vp]
    lib.fenerf_rays_workspace_bytes.restype = sz
    lib.fenerf_rays_workspace_bytes.argtypes = [P(RenderDesc), P(FieldDesc), i32]
    lib.fenerf_rays_workspace_layout.restype = C.c_int
    lib.fenerf_rays_workspace_layout.argtypes = [P(RenderDesc), P(FieldDesc), i32, P(RaysWorkspaceOffsets)]
    lib.fenerf_render_rays_grad.restype = C.c_int
    lib.fenerf_render_rays_grad.argtypes = [P(RenderDesc), P(FieldDesc), vp, vp, vp, vp, i32] + [vp] * 9 + [vp, sz, vp]
    lib.fenerf_rays_grad_workspace_layout.restype = C.c_int
    lib.fenerf_rays_grad_workspace_layout.argtypes = [P(RenderDesc), P(FieldDesc), i32, P(RaysWorkspaceOffsets), P(sz)]
    lib.fenerf_composite_backward_rays_dz.restype = C.c_int
    lib.fenerf_composite_backward_rays_dz.argtypes = [P(RenderDesc), i32] + [vp] * 7
    lib.fenerf_grid_coord_grad.restype = C.c_int
    lib.fenerf_grid_coord_grad.argtypes = [P(FieldDesc), vp, vp, vp, i32, i64, vp, i32, vp]
    lib.fenerf_ray_dir_grad.restype = C.c_int
    lib.fenerf_ray_dir_grad.argtypes = [i64, i32, i32, vp, vp, vp, vp, vp, vp]
    lib.fenerf_composite_backward_rays.restype = C.c_int
    lib.fenerf_composite_backward_rays.argtypes = [P(RenderDesc), i32] + [vp] * 9
    lib.fenerf_composite_backward.restype = C.c_int
    lib.fenerf_composite_backward.argtypes = [P(RenderDesc), i32] + [vp] * 9
    lib.fenerf_film_forward_stash.restype = C.c_int
    lib.fenerf_film_forward_stash.argtypes = [vp, vp, vp, i64, i64, i64, vp, i32, vp, vp, vp, i32, vp]
    lib.fenerf_gate_backward.restype = C.c_int
    lib.fenerf_gate_backward.argtypes = [vp, vp, i64, i64, vp, i32, vp]
    lib.fenerf_head_grads.restype = C.c_int
    lib.fenerf_head_grads.argtypes = [vp, vp, i64, i32, i32, vp, vp, vp, i32, vp]
    lib.fenerf_extras_gather.restype = C.c_int
    lib.fenerf_extras_gather.argtypes = [P(FieldDesc), vp, vp, vp, i64, i64, i32, i32, vp, vp]
    lib.fenerf_grid_scatter_add.restype = C.c_int
    lib.fenerf_grid_scatter_add.argtypes = [P(FieldDesc), vp, vp, i32, i64, vp, i32, vp]
    lib.fenerf_grid_unpack_grad.restype = C.c_int
    lib.fenerf_grid_unpack_grad.argtypes = [P(FieldDesc), vp, vp, vp, vp]
    lib.fenerf_gate_backward_det.restype = C.c_int
    lib.fenerf_gate_backward_det.argtypes = [vp, vp, i64, i64, vp, sz, vp, i32, vp]
    lib.fenerf_absmax_finite.restype = C.c_int
    lib.fenerf_absmax_finite.argtypes = [vp, i64, i32, i64, i32, vp, vp]
    lib.fenerf_grid_scatter_det_workspace_bytes.restype = sz
    lib.fenerf_grid_scatter_det_workspace_bytes.argtypes = [P(FieldDesc)]
    lib.fenerf_grid_scatter_add_det.restype = C.c_int
    lib.fenerf_grid_scatter_add_det.argtypes = [P(FieldDesc), vp, vp, i32, i64, vp, sz, vp, i32, vp]
    lib.fenerf_det_launch_count.restype = i64
    lib.fenerf_det_launch_count.argtypes = []
    lib.fenerf_gemm_nt_f16.restype = C.c_int
    lib.fenerf_gemm_nt_f16.argtypes = [vp, vp, i64, vp, vp, vp, vp]
    lib.fenerf_gemm_nt_film.restype = C.c_int
    lib.fenerf_gemm_nt_film.argtypes = [vp, vp, i64, vp, vp, i64, i64, vp, vp, vp, vp, vp]
    lib.fenerf_gemm_tn_f16.restype = C.c_int
    lib.fenerf_gemm_tn_f16.argtypes = [vp, vp, i32, i64, i32, vp, vp, vp]
    lib.fenerf_gemm_nt_split.restype = C.c_int
    lib.fenerf_gemm_nt_split.argtypes = [vp, vp, vp, i64, vp, vp, vp, vp]
    lib.fenerf_gemm_nt_film_split.restype = C.c_int
    lib.fenerf_gemm_nt_film_split.argtypes = [vp, vp, vp, i64, vp, vp, vp, i64, i64, vp, vp, vp]
    lib.fenerf_gemm_tn_split.restype = C.c_int
    lib.fenerf_gemm_tn_split.argtypes = [vp, vp, i32, i64, i32, vp, vp, vp, vp]
    lib.fenerf_absmax_f32.restype = C.c_int
    lib.fenerf_absmax_f32.argtypes = [vp, i64, vp, vp]
    lib.fenerf_debug_stage_times.restype = C.c_int
    lib.fenerf_debug_stage_times.argtypes = [i32, vp]
    lib.fenerf_debug_fast_variant.restype = C.c_int
    lib.fenerf_debug_fast_variant.argtypes = [i32, vp, i32]
    lib.fenerf_debug_soft_sine.restype = C.c_int
    lib.fenerf_debug_soft_sine.argtypes = [vp, vp, i64, vp]
    lib.fenerf_guard_stats.restype = C.c_int
    lib.fenerf_guard_stats.argtypes = [vp, P(GuardReport), vp]
    lib.fenerf_mapping_film.restype = C.c_int
    lib.fenerf_mapping_film.argtypes = [P(MappingParams), vp, i32, i32, i32, i32, vp, vp, C.c_float, vp, vp, vp]
    lib.fenerf_mask2color.restype = C.c_int
    lib.fenerf_mask2color.argtypes = [vp, i32, i32, i64, vp, vp]
    lib.fenerf_frames_to_u8.restype = C.c_int
    lib.fenerf_frames_to_u8.argtypes = [vp, i32, i32, i32, i32, i64, vp, vp]
    lib.fenerf_mc_workspace_bytes.restype = sz
    lib.fenerf_mc_workspace_bytes.argtypes = [i32]
    lib.fenerf_mc_count.restype = C.c_int
    lib.fenerf_mc_count.argtypes = [vp, i32, C.c_float, vp, sz, vp, vp]
    lib.fenerf_mc_emit.restype = C.c_int
    lib.fenerf_mc_emit.argtypes = [vp, i32, C.c_float, P(C.c_float), C.c_float, vp, sz, i64, i64, vp, vp, vp]
    lib.fenerf_last_error.restype = C.c_char_p
    lib.fenerf_last_error.argtypes = []
    lib.fenerf_abi_version.restype = i32
    lib.fenerf_abi_version.argtypes = []
    lib.fenerf_launch_count.restype = i64
    lib.fenerf_launch_count.argtypes = []


def lib():
    """The loaded library. Raises (never falls back) if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libfenerf_b200.so is missing (%s): run `python -m fenerf_b200.build` or "
                "__graft_entry__.build(); the render path has no CPU / PyTorch fallback" % LIB_PATH)
        handle = C.CDLL(LIB_PATH)
        _declare(handle)
        if handle.fenerf_abi_version() != ABI_VERSION:
            raise RuntimeError("libfenerf_b200.so ABI version mismatch")
        _lib = handle
    return _lib


class FenerfError(RuntimeError):
    def __init__(self, code, message):
        super().__init__("fenerf_b200 error %d: %s" % (code, message))
        self.code = code


def check(code):
    if code != 0:
        msg = lib().fenerf_last_error().decode("utf-8", "replace")
        if code == E_CLAMP_MODE:
            # the reference does `raise "Need to choose clamp mode"`, a TypeError in python 3
            # (generators/volumetric_rendering.py:33-34)
            raise TypeError("exceptions must derive from BaseException")
        raise FenerfError(code, msg)


def launch_count():
    return int(lib().fenerf_launch_count())


def det_launch_count():
    """Kernels launched by the deterministic backward's entries (the *_det ones) since load."""
    return int(lib().fenerf_det_launch_count())
