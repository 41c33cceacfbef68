"""ctypes binding of include/vqvae_b200.h (the C-ABI boundary).

The library is built in-tree by vqvae_b200/build.py (nvcc, sm_90a).  Loading never
falls back to anything: if the shared object is missing the import of the product
fails loudly.
"""
import ctypes as C
import os

from .build import LIB, build

_lib = None

# enums of include/vqvae_b200.h
NCHW, NHWC = 0, 1
FP32, TF32, BF16 = 0, 1, 2
PRECISIONS = {"fp32": FP32, "tf32": TF32, "bf16": BF16}
# enum vqb_status: the shape is outside what the kernels implement
ERR_UNSUPPORTED = -2
# enum vqb_conv_kind
CONV_K1, CONV_K3, CONVT_K3, CONV_K4S2, CONVT_K4S2, CONVT_K4S2_OUT, RES_W2 = range(7)

_vp, _i, _i64, _sz, _f = C.c_void_p, C.c_int, C.c_int64, C.c_size_t, C.c_float

# name -> (restype, argtypes); mirrors the header one to one (tests check this)
SIGNATURES = {
    "vqb_abi_version": (_i, []),
    "vqb_diag_build": (_i, []),
    "vqb_error_string": (C.c_char_p, [_i]),
    "vqb_device_info": (_i, [C.POINTER(_i)] * 3),
    "vqb_pack_conv_weight_f32": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "vqb_conv2d_f32": (_i, [_vp] * 5 + [_i] * 14 + [_vp]),
    "vqb_vq_workspace_bytes": (_sz, [_i64, _i, _i]),
    "vqb_vq_forward_f32": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "vqb_memcpy_async": (_i, [_vp, _vp, _sz, _i, _vp]),
    "vqb_vq_finish_f32": (_i, [_vp, _vp, _i64, _i, _i, _f, _vp, _vp, _vp]),
    "vqb_vq_backward_f32": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _f, _vp, _vp, _vp]),
    "vqb_vq_ema_workspace_bytes": (_sz, [_i64, _i, _i]),
    "vqb_vq_ema_update_f32": (_i, [_vp, _vp, _vp, _i64, _i, _i, _f, _f, _vp, _vp, _vp, _vp, _sz, _vp]),
    "vqb_vq_ema_restart_workspace_bytes": (_sz, [_i64, _i]),
    "vqb_vq_ema_restart_f32": (_i, [_vp, _vp, _i64, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "vqb_vq_commit_backward_f32": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _f, _vp, _vp]),
    "vqb_vq_finish_ema_f32": (_i, [_vp, _vp, _i64, _i, _i, _f, _vp, _vp, _vp]),
    "vqb_onehot_f32": (_i, [_vp, _i64, _i, _vp, _vp]),
    "vqb_gather_rows_f32": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp]),
    "vqb_nchw_to_nhwc_f32": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "vqb_nhwc_to_nchw_f32": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "vqb_relu_f32": (_i, [_vp, _i64, _vp]),
    "vqb_launch_count": (C.c_ulonglong, []),
    "vqb_set_vq_kernel": (_i, [_i]),
    "vqb_residual_layer_f32": (_i, [_vp] * 5 + [_i] * 7 + [_vp]),
    "vqb_residual_stack_f32": (_i, [_vp] * 6 + [_i] * 7 + [_vp]),
    "vqb_latent_block_tf32": (_i, [_vp] * 3 + [_i] + [_vp] * 2 + [_i] + [_vp] * 2 + [_i, _vp] + [_i] * 6 + [_vp]),
    "vqb_latent_block_supported": (_i, [_i] * 6),
    "vqb_decoder_tail_tf32": (_i, [_vp] * 7 + [_i] * 7 + [_vp]),
    "vqb_decoder_tail_supported": (_i, [_i] * 5),
    "vqb_conv_bf16_packed_bytes": (_sz, [_i, _i, _i]),
    "vqb_pack_conv_weight_bf16": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "vqb_conv2d_bf16": (_i, [_vp, _vp, _vp, _vp] + [_i] * 8 + [_vp]),
    "vqb_conv_in_bf16": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "vqb_vq_forward_bf16zq_f32": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "vqb_residual_layer_bf16": (_i, [_vp] * 4 + [_i] * 6 + [_vp]),
    "vqb_debug_vq_scores_f32": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    "vqb_prior_pack_f32": (_i, [_vp, _vp] + [_i] * 6 + [_vp]),
    "vqb_prior_workspace_bytes": (_sz, [_i] * 6),
    "vqb_prior_gate_f32": (_i, [_vp, _vp, _i64, _i, _i64, _vp]),
    "vqb_prior_layer_f32": (_i, [_vp] * 4 + [_i] * 5 + [_vp] * 4),
    "vqb_prior_forward_f32": (_i, [_vp] * 3 + [_i] * 3 + [_vp, _vp, _sz, _vp]),
    "vqb_prior_generate_f32": (_i, [_vp] * 3 + [_i] * 3 + [_vp] * 3 + [_sz, _vp]),
    "vqb_prior_complete_workspace_bytes": (_sz, [_i] * 6),
    "vqb_prior_complete_f32": (_i, [_vp] * 4 + [_i64] + [_i] * 3 + [_vp] * 3 + [_sz, _vp]),
    "vqb_prior_sample_workspace_bytes": (_sz, [_i] * 6 + [_i64]),
    "vqb_prior_sample_f32": (_i, [_vp] * 4 + [_i64] + [_i] * 3 + [_vp] * 5 + [_sz, _vp]),
    "vqb_prior_train_saved_bytes": (_sz, [_i] * 5),
    "vqb_prior_forward_train_f32": (_i, [_vp] * 3 + [_i] * 3 + [_vp, _vp, _sz, _vp]),
    "vqb_prior_backward_workspace_bytes": (_sz, [_vp] + [_i] * 3),
    "vqb_prior_backward_f32": (_i, [_vp] * 3 + [_i] * 3 + [_vp] * 4 + [_sz, _vp]),
    "vqb_prior_gate_backward_f32": (_i, [_vp] * 3 + [_i64, _i, _i64, _vp]),
    "vqb_prior_layer_train_saved_bytes": (_sz, [_i] * 4),
    "vqb_prior_layer_forward_train_f32": (_i, [_vp] * 4 + [_i] * 5 + [_vp] * 4 + [_sz, _vp]),
    "vqb_prior_layer_backward_workspace_bytes": (_sz, [_vp] + [_i] * 5),
    "vqb_prior_layer_backward_f32": (_i, [_vp] * 4 + [_i] * 5 + [_vp] * 7 + [_sz, _vp]),
    "vqb_prior_workspace_bytes_tf32": (_sz, [_i] * 6),
    "vqb_prior_forward_tf32": (_i, [_vp] * 3 + [_i] * 3 + [_vp, _vp, _sz, _vp]),
    "vqb_prior_forward_train_tf32": (_i, [_vp] * 3 + [_i] * 3 + [_vp, _vp, _sz, _vp]),
    "vqb_prior_backward_tf32": (_i, [_vp] * 3 + [_i] * 3 + [_vp] * 4 + [_sz, _vp]),
    "vqb_prior_log_prob_workspace_bytes": (_sz, [_i] * 6),
    "vqb_prior_log_prob_workspace_bytes_tf32": (_sz, [_i] * 6),
    "vqb_prior_log_prob_f32": (_i, [_vp] * 3 + [_i64] + [_i] * 3 + [_vp] * 3 + [_sz, _vp]),
    "vqb_prior_log_prob_tf32": (_i, [_vp] * 3 + [_i64] + [_i] * 3 + [_vp] * 3 + [_sz, _vp]),
    "vqb_relu_backward_f32": (_i, [_vp, _vp, _vp, _i64, _vp]),
    "vqb_conv_wgrad_workspace_bytes": (_sz, [_i] * 10),
    "vqb_conv_wgrad_f32": (_i, [_vp] * 4 + [_i] * 12 + [_vp, _sz, _vp]),
    "vqb_adam_capacity": (_i, []),
    "vqb_adam_multi_f32": (_i, [_vp, _i] + [C.c_double] * 5 + [_i, _vp]),
    "vqb_repack_capacity": (_i, []),
    "vqb_repack_multi": (_i, [_vp, _i, _vp, _i, _vp]),
}

PRIOR_MAX_LAYERS = 32       # VQB_PRIOR_MAX_LAYERS
PRIOR_MAX_KERNEL = 15       # VQB_PRIOR_MAX_KERNEL


class PriorLayerWeights(C.Structure):
    """struct vqb_prior_layer_weights"""
    _fields_ = [(n, _vp) for n in ("vert_w", "vert_b", "v2h_w", "v2h_b", "horiz_w", "horiz_b", "resid_w", "resid_b",
                                   "class_emb")] + [("kernel", _i), ("mask_a", _i), ("residual", _i)]


class PriorNet(C.Structure):
    """struct vqb_prior_net"""
    _fields_ = [("layers", C.POINTER(PriorLayerWeights)), ("n_layers", _i), ("embedding", _vp), ("out1_w", _vp),
                ("out1_b", _vp), ("out2_w", _vp), ("out2_b", _vp), ("input_dim", _i), ("dim", _i), ("n_classes", _i)]


class PriorSampling(C.Structure):
    """struct vqb_prior_sampling"""
    _fields_ = [("temperature", _f), ("top_k", _i), ("top_p", _f)]


class PriorLayerGrads(C.Structure):
    """struct vqb_prior_layer_grads"""
    _fields_ = [(n, _vp) for n in ("vert_w", "vert_b", "v2h_w", "v2h_b", "horiz_w", "horiz_b", "resid_w", "resid_b",
                                   "class_emb")]


class PriorGrads(C.Structure):
    """struct vqb_prior_grads"""
    _fields_ = [("layers", C.POINTER(PriorLayerGrads)), ("n_layers", _i), ("embedding", _vp), ("out1_w", _vp),
                ("out1_b", _vp), ("out2_w", _vp), ("out2_b", _vp)]


# enum vqb_pack_layout
PACK_F32, PACK_SHUFFLE_F32, PACK_BF16, PACK_SHUFFLE_BF16, PACK_PRIOR_F32, PACK_MASK_ZERO = range(6)


class AdamTensor(C.Structure):
    """struct vqb_adam_tensor"""
    _fields_ = [(n, _vp) for n in ("param", "grad", "exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step")] + \
        [("numel", _i64)]


class PackDesc(C.Structure):
    """struct vqb_pack_desc"""
    _fields_ = [("dst", _vp), ("src", _vp)] + [(n, _i) for n in ("layout", "Cout", "Cin", "Cin_pad", "kh", "kw",
                                                                 "transposed", "rows", "cols")]


def lib():
    """The loaded C-ABI library (built on first use if the .so is absent/stale)."""
    global _lib
    if _lib is None:
        path = LIB if os.path.exists(LIB) and os.environ.get("VQB_NO_REBUILD") else build()
        handle = C.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)   # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        if handle.vqb_abi_version() != 3:
            raise RuntimeError("libvqvae_b200.so ABI version mismatch")
        _lib = handle
    return _lib


def check(code, what):
    if code != 0:
        msg = lib().vqb_error_string(int(code)).decode()
        raise RuntimeError(f"{what}: {msg} (code {code})")
