"""ctypes binding of libvqb200.so (the C ABI declared in include/vqb200.h).

There is NO fallback: if the library cannot be loaded (or built) importing this module raises, and
every op raises on non-CUDA tensors.  PyTorch is used only for device memory and streams.
"""
import ctypes
import os

from . import build as _build

_c = ctypes
_i32, _i64, _f32, _f64, _vp, _sz = _c.c_int, _c.c_int64, _c.c_float, _c.c_double, _c.c_void_p, _c.c_size_t

DTYPE_F32, DTYPE_BF16 = 0, 1
METRIC_EUCLID, METRIC_COSINE = 0, 1
VQB_LQ_MAX_DIM, VQB_LQ_MAX_VALUES = 256, 8192   # LatentQuantize's table cap (include/vqb200.h)

class FusedOutputs(ctypes.Structure):
    """Mirror of `vqb_fused_outputs` (include/vqb200.h)."""
    _fields_ = [("x_eff", _vp), ("embed", _vp), ("q_out", _vp), ("idx64_out", _vp), ("idx_stride", _i64),
                ("loss_sum", _vp), ("x_raw", _vp), ("resid_out", _vp), ("qsum", _vp), ("stats_cnt", _vp), ("stats_sum", _vp),
                ("dtype", _i32), ("planes_out", _vp)]


class VQForwardArgs(ctypes.Structure):
    """Mirror of `vqb_vq_forward_args` (include/vqb200.h)."""
    _fields_ = [("x", _vp), ("dtype", _i32), ("metric", _i32), ("N", _i64), ("D", _i32), ("K", _i32),
                ("already_normalised", _i32), ("cluster_size", _vp), ("embed_avg", _vp), ("embed", _vp),
                ("planes", _vp), ("bext", _vp), ("bias", _vp), ("cnorm2", _vp), ("cmax", _vp), ("scratch", _vp),
                ("q_out", _vp), ("idx64_out", _vp), ("idx_stride", _i64), ("loss_out", _vp), ("loss_weight", _f32),
                ("resid_out", _vp), ("qsum", _vp), ("idx32", _vp), ("update", _i32), ("stats_mode", _i32), ("stats_accumulate", _i32), ("do_normalise", _i32),
                ("decay", _f64), ("eps", _f64), ("stats", _vp), ("margin_rel", _f32), ("workspace", _vp),
                ("workspace_bytes", _sz), ("ev_search_begin", _vp), ("ev_search_end", _vp),
                ("peer_stats", _vp), ("peer_flags", _vp), ("peer_epoch", _vp), ("peer_rank", _i32), ("peer_world", _i32),
                ("peer_slice_offset", _i64), ("a_planes_in", _vp), ("planes_out", _vp), ("row_mask", _vp), ("n_live", _vp)]


class RvqEmaArgs(ctypes.Structure):
    _fields_ = [("cluster_size", _vp), ("embed_avg", _vp), ("embed", _vp), ("stats", _vp), ("K", _i32), ("D", _i32),
                ("decay", _f64), ("eps", _f64), ("metric", _i32), ("do_lerp", _i32), ("do_normalise", _i32),
                ("planes", _vp), ("bext", _vp), ("bias", _vp), ("cnorm2", _vp), ("cmax", _vp), ("scratch", _vp),
                ("n_lerp", _i32), ("slice_stride", _i64)]


class RvqAccArgs(ctypes.Structure):
    _fields_ = [("embeds", _vp), ("embed_stride", _i64), ("Q", _i32), ("K", _i32), ("D", _i32), ("idx", _vp), ("N", _i64),
                ("out", _vp), ("dtype", _i32)]


class RvqBarArgs(ctypes.Structure):
    _fields_ = [("flags", _vp), ("epoch", _vp), ("rank", _i32), ("world", _i32)]


class RvqEmaPeersArgs(ctypes.Structure):
    _fields_ = [("cluster_size", _vp), ("embed_avg", _vp), ("embed", _vp), ("peer_stats", _vp), ("slice_offset", _i64),
                ("world", _i32), ("K", _i32), ("D", _i32), ("decay", _f64), ("eps", _f64), ("metric", _i32),
                ("do_normalise", _i32), ("planes", _vp), ("bext", _vp), ("bias", _vp), ("cnorm2", _vp), ("cmax", _vp),
                ("scratch", _vp), ("n_lerp", _i32), ("slice_stride", _i64)]


class RvqSimvqArgs(ctypes.Structure):
    _fields_ = [("r", _vp), ("codes", _vp), ("idx", _vp), ("N", _i64), ("D", _i32), ("rotation", _i32), ("r_next", _vp),
                ("qsum", _vp), ("first", _i32), ("idx64_out", _vp), ("idx_stride", _i64), ("loss_sum", _vp), ("loss_out", _vp),
                ("input_weight", _f32), ("weight", _f32)]


class RvqOp(ctypes.Structure):
    """Mirror of `vqb_rvq_op` (include/vqb200.h)."""
    _fields_ = [("kind", _i32), ("lane", _i32), ("stage", VQForwardArgs), ("ema", RvqEmaArgs), ("acc", RvqAccArgs),
                ("bar", RvqBarArgs), ("emap", RvqEmaPeersArgs), ("simvq", RvqSimvqArgs)]


RVQ_STAGE, RVQ_EMA, RVQ_ACCUMULATE, RVQ_BARRIER, RVQ_EMA_PEERS, RVQ_SIMVQ_TAIL = 0, 1, 2, 3, 4, 5

SIGNATURES = {
    "vqb_version": (_i32, []),
    "vqb_strerror": (_c.c_char_p, [_i32]),
    "vqb_padded_codes": (_i32, [_i32]),
    "vqb_codebook_prepare": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqb_input_prepare": (_i32, [_vp, _i32, _i64, _i32, _i32, _vp, _vp, _i32, _vp]),
    "vqb_assign": (_i32, [_vp, _i32, _i64, _i32, _vp, _vp, _vp, _i32, _f32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqb_assign_ex": (_i32, [_vp, _i32, _i64, _i32, _vp, _vp, _vp, _i32, _f32, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp]),
    "vqb_fix_flagged": (_i32, [_vp, _i32, _i64, _i32, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "vqb_gather": (_i32, [_vp, _i32, _i64, _i32, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "vqb_loss_finalize": (_i32, [_vp, _i64, _i32, _f32, _vp, _vp]),
    "vqb_stats_offset": (_i64, [_i32]),
    "vqb_stats_floats": (_i64, [_i32, _i32]),
    "vqb_ema_stats_workspace": (_sz, [_i64, _i32]),
    "vqb_ema_stats": (_i32, [_vp, _i32, _i64, _i32, _vp, _i32, _vp, _vp, _sz, _vp]),
    "vqb_ema_apply": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _f64, _f64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqb_rotate": (_i32, [_vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp]),
    "vqb_rotate_masked": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _f32, _i32, _i32, _i64, _i32, _i32, _vp, _vp]),
    "vqb_diveq": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _f32, _vp, _vp, _vp]),
    "vqb_peer_barrier": (_i32, [_vp, _i32, _i32, _vp, _vp]),
    "vqb_ema_apply_peers": (_i32, [_vp, _vp, _vp, _vp, _i32, _i64, _i32, _i32, _f64, _f64, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqb_ema_apply_weighted": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _f64, _f64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqb_vq_forward_workspace": (_sz, [_i64, _i32, _i32, _i32, _i32, _i32]),
    "vqb_vq_forward": (_i32, [_vp, _vp]),
    "vqb_debug_set_profile_buffer": (_i32, [_vp]),
    "vqb_debug_set_mode": (_i32, [_i32]),
    "vqb_debug_active": (_i32, []),
    "vqb_debug_graph_stats": (_i32, [_vp]),
    "vqb_debug_assign_plan": (_i32, [_i32, _i32, _i32, _vp]),
    "vqb_debug_stats_plan": (_i32, [_i64, _i32, _i32, _vp]),
    "vqb_decode": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _i64, _vp, _i32, _vp]),
    "vqb_rvq_accumulate": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _i64, _vp, _i32, _vp]),
    "vqb_debug_gather_sum_plan": (_i32, [_i32, _i32, _i32, _i32, _i64, _i32, _vp]),
    "vqb_rvq_forward": (_i32, [_vp, _i32, _vp]),
    "vqb_rsimvq_tail": (_i32, [_vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp, _i32, _vp, _i64, _vp, _vp, _f32, _f32, _vp]),
    "vqb_rsimvq_backward": (_i32, [_vp, _vp, _i32, _i32, _vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "vqb_fsq_forward": (_i32, [_vp, _i32, _i32, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _i64,
                               _i64, _vp]),
    "vqb_fsq_backward": (_i32, [_vp, _i32, _i32, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqb_fsq_decode": (_i32, [_vp, _i32, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqb_lfq_forward": (_i32, [_vp, _i32, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp,
                               _vp, _i32, _vp]),
    "vqb_lfq_forward_blocks": (_i32, [_i64, _i32]),
    "vqb_lfq_entropy": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _i64, _i64, _vp, _f32, _i32, _vp, _vp, _vp]),
    "vqb_lfq_entropy_tiles": (_i32, [_i32]),
    "vqb_lfq_entropy_backward": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _i64, _i64, _vp, _f32, _vp, _vp, _i32, _vp, _vp, _vp]),
    "vqb_lfq_backward": (_i32, [_vp, _i32, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqb_lfq_decode": (_i32, [_vp, _i32, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "vqb_fsp_blocks": (_i32, [_i64]),
    "vqb_fsp_forward": (_i32, [_vp, _i32, _i64, _i32, _i32, _i32, _vp, _f32, _vp, _vp, _f32, _f32, _f32, _vp, _vp, _vp, _vp, _i32,
                               _vp]),
    "vqb_fsp_stats": (_i32, [_vp, _i32, _i64, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp]),
    "vqb_fsp_backward": (_i32, [_vp, _i32, _i64, _i32, _i32, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqb_fsp_decode": (_i32, [_vp, _i32, _i64, _i32, _i32, _i32, _vp, _f32, _f32, _vp, _vp, _vp]),
    "vqb_binmap_hot": (_i32, [_vp, _vp, _i64, _i32, _vp, _vp]),
    "vqb_binmap_backward_plan": (_i32, [_i64, _i32, _i32, _vp]),
    "vqb_binmap_backward": (_i32, [_vp, _i64, _i32, _vp, _i64, _i64, _i32, _vp, _vp, _vp]),
    "vqb_hvq_pool": (_i32, [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp]),
    "vqb_hvq_pool_backward": (_i32, [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp]),
    "vqb_hvq_upsample": (_i32, [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vqb_hvq_upsample_backward": (_i32, [_vp, _vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp]),
    "vqb_hvq_blend_update": (_i32, [_vp, _vp, _i64, _f64, _vp, _vp, _vp, _vp, _vp]),
    "vqb_hvq_blend_backward": (_i32, [_vp, _vp, _i64, _f64, _vp, _vp, _vp]),
    "vqb_rpq_norm_project": (_i32, [_vp, _i64, _i32, _vp, _i32, _i32, _i32, _vp, _vp]),
    "vqb_lq_quantize": (_i32, [_vp, _i32, _i64, _i32, _i32, _vp, _i32, _vp, _vp, _vp, _vp]),
    "vqb_lq_loss_blocks": (_i32, [_i64]),
    "vqb_lq_loss": (_i32, [_vp, _i32, _vp, _i64, _vp, _vp, _i32, _i32, _vp, _i32, _vp, _vp]),
    "vqb_lq_loss_backward": (_i32, [_vp, _i32, _vp, _i64, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp]),
}


def _load():
    path = os.environ.get("VQB200_LIB")
    if not path:
        path = _build.LIB
        if _build.is_stale():
            if _build.find_nvcc() is not None:
                path = _build.build()
            elif not os.path.exists(path):
                raise ImportError("vqb200: libvqb200.so is missing and nvcc is not available to build it; "
                                  "run `python -m vector_quantize_pytorch_b200.build` where nvcc exists")
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export the symbol
        fn.restype = res
        fn.argtypes = args
    return lib, path


lib, LIB_PATH = _load()


class VQBError(RuntimeError):
    pass


def check(rc, what):
    if rc != 0:
        raise VQBError(f"{what}: {lib.vqb_strerror(rc).decode()} (code {rc})")
