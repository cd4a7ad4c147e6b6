"""ctypes binding of libddn_b200.so (the C ABI declared in include/ddn_b200.h).

There is no CPU or PyTorch fallback: if the library cannot be loaded, importing this module raises.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libddn_b200.so")

PRECISION_FP32_SIMT, PRECISION_BF16X3, PRECISION_BF16 = 0, 1, 2
MODE_INFER, MODE_TRAIN, MODE_EVAL_SAVE = 0, 1, 2
ARCH_RESNET34_8S, ARCH_RESNET50_8S = 0, 1
GRAD_BUCKET_FN = ctypes.CFUNCTYPE(None, ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int64)
TERM_MATCH, TERM_HINGE, TERM_HINGE_INV = 0, 1, 2
TERM_PIXEL_WEIGHT = 1
NET_UNIT_DESCRIPTORS = 1     # ddn_net_*_v2 flags: unit-length descriptors (the reference's `normalize`, per pixel)
LOWRES_UNIT = 1              # ddn_contrastive_terms_*_lowres_v2 flags: the sampled descriptors are normalised to unit length
MAX_TERMS = 8

c_f32p = ctypes.POINTER(ctypes.c_float)
vp, i32, i64, f32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_size_t


class TensorEntry(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char * 64), ("ndim", ctypes.c_int32), ("shape", ctypes.c_int32 * 4),
                ("offset", ctypes.c_int64), ("numel", ctypes.c_int64)]


class LossTerm(ctypes.Structure):
    _fields_ = [("idx_a", vp), ("idx_b", vp), ("gt_b", vp), ("n", i64), ("n_gt", i64),
                ("kind", ctypes.c_int32), ("flags", ctypes.c_int32), ("margin", f32), ("m_pixel", f32),
                ("len", vp), ("len_gt", vp)]


class ProfileEntry(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char * 32), ("launches", ctypes.c_int64), ("ms", ctypes.c_double), ("work", ctypes.c_double)]


class WithinSceneCfg(ctypes.Structure):
    _fields_ = [("match_loss_weight", f32), ("non_match_loss_weight", f32),
                ("scale_by_hard_negatives", ctypes.c_int32), ("has_blind", ctypes.c_int32),
                ("n_match", i64), ("n_masked", i64), ("n_background", i64), ("n_blind", i64),
                ("len_match", vp), ("len_masked", vp), ("len_background", vp), ("len_blind", vp)]


class PairTypeComposeCfg(ctypes.Structure):
    _fields_ = [("match_loss_weight", f32), ("non_match_loss_weight", f32),
                ("scale_by_hard_negatives", ctypes.c_int32), ("scale_by_hard_negatives_different_object", ctypes.c_int32),
                ("n_match", i64), ("n_masked", i64), ("n_background", i64), ("n_blind", i64),
                ("len_match", vp), ("len_masked", vp), ("len_background", vp), ("len_blind", vp)]


class WsBatchCfg(ctypes.Structure):
    _fields_ = [("B", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
                ("sample_matches_only_off_mask", ctypes.c_int32), ("domain_randomize", ctypes.c_int32),
                ("use_image_b_mask_inv", ctypes.c_int32), ("n_attempts", i64), ("k_masked", i64), ("k_background", i64),
                ("mean", f32 * 3), ("std", f32 * 3)]


class WsBatchRand(ctypes.Structure):
    _fields_ = [(k, vp) for k in ("params", "noise", "cand_u", "cand_v", "masked_u", "masked_v", "background_u",
                                  "background_v", "blind")]


class WsBatchOut(ctypes.Structure):
    _fields_ = [(k, vp) for k in ("image_a", "image_b", "matches_a", "matches_b", "masked_a", "masked_b", "background_a",
                                  "background_b", "blind_a", "blind_b", "counts", "empty")]


WS_MAX_PAIRS = 128
WS_RANDOMIZE, WS_GRADIENT, WS_VERTICAL, WS_NOISE, WS_FLIP, WS_RGB1, WS_RGB2, WS_PARAM_BYTES = 0, 1, 2, 3, 4, 5, 8, 16


class AsBatchCfg(ctypes.Structure):
    _fields_ = [("B", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32), ("domain_randomize", ctypes.c_int32),
                ("num_samples", i64), ("mean", f32 * 3), ("std", f32 * 3)]


class AsBatchRand(ctypes.Structure):
    _fields_ = [(k, vp) for k in ("params", "noise", "blind_a", "blind_b")]


class AsBatchOut(ctypes.Structure):
    _fields_ = [(k, vp) for k in ("image_a", "image_b", "blind_a", "blind_b", "counts", "empty")]


AS_MAX_PAIRS = 16384


class SmoBatchCfg(ctypes.Structure):
    _fields_ = [("B", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
                ("sample_matches_only_off_mask", ctypes.c_int32), ("use_image_b_mask_inv", ctypes.c_int32),
                ("n_attempts", i64), ("k_masked", i64), ("k_background", i64), ("mean", f32 * 3), ("std", f32 * 3)]


class SmoBatchRand(ctypes.Structure):
    _fields_ = [(k, vp) for k in ("merge", "cand_u", "cand_v", "masked_u", "masked_v", "background_u", "background_v")]


class SmoBatchOut(ctypes.Structure):
    _fields_ = [(k, vp) for k in ("image_a", "image_b", "matches_a", "matches_b", "masked_a", "masked_b", "background_a",
                                  "background_b", "blind_a", "blind_b", "counts", "empty")]


SMO_MAX_PAIRS = WS_MAX_PAIRS // 2
FRAMES_MAX_PAIRS = 128

_SIGNATURES = {
    "ddn_abi_version": (i32, []),
    "ddn_set_reserved_sms": (i32, [i32]),
    "ddn_last_error": (ctypes.c_char_p, []),
    "ddn_kernel_launch_count": (i64, []),
    "ddn_resnet34_8s_param_table": (i32, [i32, ctypes.POINTER(TensorEntry), i32]),
    "ddn_resnet34_8s_buffer_table": (i32, [ctypes.POINTER(TensorEntry), i32]),
    "ddn_resnet34_8s_param_count": (i64, [i32]),
    "ddn_resnet34_8s_buffer_count": (i64, []),
    "ddn_resnet34_8s_workspace_bytes": (sz, [i32, i32, i32, i32, i32, i32]),
    "ddn_resnet34_8s_weight_cache_bytes": (sz, [i32]),
    "ddn_resnet34_8s_set_weight_cache": (i32, [vp, sz, vp, ctypes.c_uint64, i32]),
    "ddn_resnet34_8s_forward": (i32, [vp, vp, vp, vp, vp, sz, i32, i32, i32, i32, i32, i32, f32, f32, i32, vp, vp]),
    "ddn_resnet34_8s_backward": (i32, [vp, vp, vp, vp, vp, sz, i32, i32, i32, i32, i32, i32, f32, i32, GRAD_BUCKET_FN, vp, vp]),
    "ddn_contrastive_terms_forward_lowres": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, ctypes.POINTER(LossTerm), i32, vp, vp, vp]),
    "ddn_contrastive_terms_backward_lowres": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, ctypes.POINTER(LossTerm), i32,
                                                    vp, vp, vp, vp, vp, vp]),
    "ddn_contrastive_terms_forward_lowres_v2": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, ctypes.POINTER(LossTerm), i32, vp, vp,
                                                      i32, vp]),
    "ddn_contrastive_terms_backward_lowres_v2": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, ctypes.POINTER(LossTerm), i32,
                                                       vp, vp, vp, vp, vp, i32, vp]),
    "ddn_resnet34_8s_grad_buckets": (i32, [i32, ctypes.POINTER(i64), i32]),
    "ddn_net_param_table": (i32, [i32, i32, ctypes.POINTER(TensorEntry), i32]),
    "ddn_net_buffer_table": (i32, [i32, ctypes.POINTER(TensorEntry), i32]),
    "ddn_net_param_count": (i64, [i32, i32]),
    "ddn_net_buffer_count": (i64, [i32]),
    "ddn_net_workspace_bytes": (sz, [i32] * 7),
    "ddn_net_weight_cache_bytes": (sz, [i32, i32]),
    "ddn_net_forward": (i32, [i32, vp, vp, vp, vp, vp, sz, i32, i32, i32, i32, i32, i32, f32, f32, i32, vp, vp]),
    "ddn_net_backward": (i32, [i32, vp, vp, vp, vp, vp, sz, i32, i32, i32, i32, i32, i32, f32, i32, GRAD_BUCKET_FN, vp, vp]),
    "ddn_net_grad_buckets": (i32, [i32, i32, ctypes.POINTER(i64), i32]),
    "ddn_net_workspace_bytes_v2": (sz, [i32] * 8),
    "ddn_net_forward_v2": (i32, [i32, vp, vp, vp, vp, vp, sz, i32, i32, i32, i32, i32, i32, f32, f32, i32, vp, i32, vp]),
    "ddn_net_backward_v2": (i32, [i32, vp, vp, vp, vp, vp, sz, i32, i32, i32, i32, i32, i32, f32, i32, i32, GRAD_BUCKET_FN, vp, vp]),
    "ddn_contrastive_terms_forward": (i32, [vp, vp, i64, i64, i64, i32, i64, i32, i32, ctypes.POINTER(LossTerm), i32, vp, vp, vp]),
    "ddn_contrastive_terms_backward": (i32, [vp, vp, i64, i64, i64, i32, i64, i32, i32, ctypes.POINTER(LossTerm), i32,
                                             vp, vp, vp, vp, vp]),
    "ddn_within_scene_compose": (i32, [vp, vp, i32, i32, ctypes.POINTER(WithinSceneCfg), vp, vp, vp]),
    "ddn_pair_type_compose": (i32, [vp, vp, i32, i32, ctypes.POINTER(PairTypeComposeCfg), vp, vp, vp, vp]),
    "ddn_within_scene_loss_host": (i32, [vp, vp, i32, i32, i32, i32, vp, vp, i64, vp, vp, i64, vp, vp, i64,
                                         f32, f32, f32, f32, i32, vp]),
    "ddn_conv2d_workspace_bytes": (sz, [i32] * 10),
    "ddn_conv2d_forward": (i32, [vp, vp, vp] + [i32] * 10 + [vp, sz, vp]),
    "ddn_conv2d_backward": (i32, [vp, vp, vp, vp, vp] + [i32] * 10 + [vp, sz, vp]),
    "ddn_conv2d_fused_workspace_bytes": (sz, [i32] * 10),
    "ddn_conv2d_bn_stats_forward": (i32, [vp] * 7 + [i32] * 10 + [f32, f32, i32, vp, sz, vp]),
    "ddn_conv2d_folded_forward": (i32, [vp] * 10 + [i32] * 10 + [f32, i32, vp, sz, vp]),
    "ddn_conv2d_backward_data_bn_stats": (i32, [vp] * 13 + [i32] * 11 + [vp, sz, vp]),
    "ddn_stem_pool_forward": (i32, [vp] * 9 + [i32] * 4 + [vp]),
    "ddn_stem_workspace_bytes": (sz, [i32] * 4),
    "ddn_stem_backward": (i32, [vp] * 15 + [i32] * 6 + [vp, sz, vp]),
    "ddn_batchnorm_workspace_bytes": (sz, [i64, i32]),
    "ddn_batchnorm_forward": (i32, [vp] * 9 + [i64, i32, i32, i32, f32, f32, vp, sz, vp]),
    "ddn_batchnorm_backward": (i32, [vp] * 10 + [i64, i32, i32, vp, sz, vp]),
    "ddn_upsample_bilinear_forward": (i32, [vp, vp, i32, i32, i32, i32, i32, vp]),
    "ddn_upsample_bilinear_backward": (i32, [vp, vp, i32, i32, i32, i32, i32, vp]),
    "ddn_upsample_bilinear_unit_forward": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, vp]),
    "ddn_upsample_bilinear_unit_backward": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]),
    "ddn_fc_workspace_bytes": (sz, [i32, i32]),
    "ddn_fc_forward": (i32, [vp] * 7 + [i64, i32, i32, i32, vp]),
    "ddn_fc_backward": (i32, [vp] * 8 + [i64, i32, i32, i32, vp, sz, vp]),
    "ddn_scale_inplace": (i32, [vp, i64, f32, vp]),
    "ddn_sample_non_matches_scratch_bytes": (sz, [i32, i32]),
    "ddn_sample_non_matches": (i32, [vp, i32, i32, vp, vp, i64, vp, i64, vp, vp, vp, sz, vp]),
    "ddn_find_pixel_correspondences_scratch_bytes": (sz, [i64]),
    "ddn_find_pixel_correspondences": (i32, [vp, vp, i32, i32, vp, i64, vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]),
    "ddn_within_scene_batch_scratch_bytes": (sz, [ctypes.POINTER(WsBatchCfg)]),
    "ddn_within_scene_batch": (i32, [ctypes.POINTER(WsBatchCfg)] + [vp] * 9 + [ctypes.POINTER(WsBatchRand),
                                     ctypes.POINTER(WsBatchOut), vp, sz, vp]),
    "ddn_across_scene_batch_scratch_bytes": (sz, [ctypes.POINTER(AsBatchCfg)]),
    "ddn_across_scene_batch": (i32, [ctypes.POINTER(AsBatchCfg)] + [vp] * 4 + [ctypes.POINTER(AsBatchRand),
                                     ctypes.POINTER(AsBatchOut), vp, sz, vp]),
    "ddn_synthetic_multi_object_batch_scratch_bytes": (sz, [ctypes.POINTER(SmoBatchCfg)]),
    "ddn_synthetic_multi_object_batch": (i32, [ctypes.POINTER(SmoBatchCfg)] + [vp] * 9 + [ctypes.POINTER(SmoBatchRand),
                                               ctypes.POINTER(SmoBatchOut), vp, sz, vp]),
    "ddn_frames_gather": (i32, [vp, vp, vp, i64, i32, i32, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp]),
    "ddn_find_best_match": (i32, [vp, i64, i64, i32, i32, i32, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp]),
    "ddn_match_statistics_scratch_bytes": (sz, [i32, i32, i32, i64]),
    "ddn_match_statistics": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, vp, vp, vp, i64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                   vp, sz, vp]),
    "ddn_best_match_batch_scratch_bytes": (sz, [i64]),
    "ddn_best_match_batch": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, vp, vp, i64, vp, vp, vp, vp, sz, vp]),
    "ddn_descriptor_statistics_scratch_bytes": (sz, [i32, i32, i32, i32]),
    "ddn_descriptor_statistics": (i32, [vp, vp, i32, i32, i32, i32, vp, i32, vp, vp, vp, sz, vp]),
    "ddn_adam_step": (i32, [vp, vp, vp, vp, i64, i64, f32, f32, f32, f32, f32, f32, vp]),
    "ddn_profile_enable": (i32, [i32]),
    "ddn_profile_reset": (i32, []),
    "ddn_profile_read": (i32, [ctypes.POINTER(ProfileEntry), i32]),
}
EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def _load():
    if not os.path.exists(LIB_PATH):
        # fresh checkout: compile the library in-tree (nvcc cross-compiles sm_90a without a GPU).  Still no fallback: if
        # nvcc is not there either, importing the package fails.
        try:
            import importlib.util
            spec = importlib.util.spec_from_file_location("_ddn_build", os.path.join(_HERE, "build.py"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            mod.build()
        except Exception as e:
            raise ImportError(
                "libddn_b200.so is missing at %s and building it failed (%s): run `python "
                "pytorch-dense-correspondence_b200/build.py`.  There is no fallback path." % (LIB_PATH, e))
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)      # AttributeError here == header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    if lib.ddn_abi_version() != 3:
        raise ImportError("libddn_b200.so ABI version mismatch")
    return lib


lib = _load()


class DdnError(RuntimeError):
    pass


def check(rc):
    if rc != 0:
        raise DdnError("libddn_b200 error %d: %s" % (rc, lib.ddn_last_error().decode()))


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda_f32(t, name, contiguous=True):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: this path has no CPU fallback" % name)
    if t.dtype != torch.float32:
        raise RuntimeError("%s must be float32 (got %s)" % (name, t.dtype))
    if contiguous and not t.is_contiguous():
        raise RuntimeError("%s must be contiguous" % name)


def param_table(D, arch=ARCH_RESNET34_8S):
    n = lib.ddn_net_param_table(arch, D, None, 0)
    check(min(n, 0))
    arr = (TensorEntry * n)()
    lib.ddn_net_param_table(arch, D, arr, n)
    return [(e.name.decode(), tuple(e.shape[:e.ndim]), int(e.offset), int(e.numel)) for e in arr]


def buffer_table(arch=ARCH_RESNET34_8S):
    n = lib.ddn_net_buffer_table(arch, None, 0)
    check(min(n, 0))
    arr = (TensorEntry * n)()
    lib.ddn_net_buffer_table(arch, arr, n)
    return [(e.name.decode(), tuple(e.shape[:e.ndim]), int(e.offset), int(e.numel)) for e in arr]


def grad_buckets(D, arch=ARCH_RESNET34_8S):
    """[(offset, numel)] of the gradient buckets in the order the backward completes them (last layers first); the count is
    the one the library reports."""
    n = lib.ddn_net_grad_buckets(arch, D, None, 0)
    check(min(n, 0))
    arr = (i64 * (n + 1))()
    lib.ddn_net_grad_buckets(arch, D, arr, n + 1)
    ends = [int(arr[n])] + [int(arr[i]) for i in range(n - 1)]
    return [(int(arr[i]), ends[i] - int(arr[i])) for i in range(n)]


NO_BUCKET_CALLBACK = ctypes.cast(None, GRAD_BUCKET_FN)


def profile_read():
    """{class name: {"launches", "ms", "flops" (conv_*) or "bytes" (loss_*)}} for the kernels timed since the last reset."""
    arr = (ProfileEntry * 16)()
    n = lib.ddn_profile_read(arr, 16)
    out = {}
    for e in arr[:n]:
        name = e.name.decode()
        out[name] = {"launches": int(e.launches), "ms": float(e.ms), ("flops" if name.startswith("conv") else "bytes"): float(e.work)}
    return out


def launch_count():
    return int(lib.ddn_kernel_launch_count())
