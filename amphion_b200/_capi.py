"""ctypes binding of libamphion_b200.so (the C ABI in include/amphion_b200.h)."""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

AB_MAX_STAGES = 8
AB_MAX_KERNELS = 8
AB_MAX_DILATIONS = 8

GEN_HIFIGAN, GEN_BIGVGAN, GEN_NSFHIFIGAN, GEN_TRUNK, GEN_MELGAN, GEN_VOCOS, GEN_DIFFWAVE, GEN_FACODEC = 0, 1, 2, 3, 4, 5, 6, 7
GEN_FACODEC_ENCODER = 8
GEN_FACODEC_REDECODER = 9
GEN_RVQ = 10
GEN_VOCOS_LINEAR = 11
AB_FACODEC_MAX_Q = 32
ACT_LRELU, ACT_SNAKE, ACT_SNAKEBETA, ACT_SNAKE1D = 0, 1, 2, 3
PRECISIONS = {"fp32": 0, "tc_f16": 1, "tc_bf16": 2}


class GeneratorConfig(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("n_mel", C.c_int32),
        ("upsample_initial_channel", C.c_int32),
        ("num_upsamples", C.c_int32),
        ("upsample_rates", C.c_int32 * AB_MAX_STAGES),
        ("upsample_kernel_sizes", C.c_int32 * AB_MAX_STAGES),
        ("resblock", C.c_int32),
        ("num_kernels", C.c_int32),
        ("resblock_kernel_sizes", C.c_int32 * AB_MAX_KERNELS),
        ("num_dilations", C.c_int32 * AB_MAX_KERNELS),
        ("resblock_dilation_sizes", (C.c_int32 * AB_MAX_DILATIONS) * AB_MAX_KERNELS),
        ("activation", C.c_int32),
        ("snake_logscale", C.c_int32),
        ("gin_channels", C.c_int32),
        ("conv_post_no_bias", C.c_int32),
        ("trunk_out_channels", C.c_int32),
        ("trunk_in_kernel", C.c_int32),
        ("trunk_out_kernel", C.c_int32),
        ("ffn_channels", C.c_int32),
        ("num_layers", C.c_int32),
        ("istft_n_fft", C.c_int32),
        ("istft_hop", C.c_int32),
        ("dilation_cycle", C.c_int32),
        ("embedding_rows", C.c_int32),
        ("vq_num_q", C.c_int32 * 3),
        ("vq_codebook_bits", C.c_int32 * 3),
        ("vq_codebook_dim", C.c_int32),
        ("facodec_quantize", C.c_int32),
        ("facodec_prosody_encoder", C.c_int32),
        ("vq_codebook_size", C.c_int32),
    ]


class ProfileEntry(C.Structure):
    _fields_ = [("name", C.c_char * 32), ("launches", C.c_int32), ("ms", C.c_float),
                ("flops", C.c_double), ("bytes", C.c_double)]


class MelConfig(C.Structure):
    _fields_ = [
        ("n_fft", C.c_int32),
        ("hop", C.c_int32),
        ("win", C.c_int32),
        ("n_mel", C.c_int32),
        ("pad", C.c_int32),
        ("eps", C.c_float),
        ("clamp", C.c_float),
    ]


# name -> (restype, argtypes); must list every symbol declared in include/amphion_b200.h
_P = C.c_void_p
_I64P = C.POINTER(C.c_int64)
SIGNATURES = {
    "ab_last_error": (C.c_char_p, []),
    "ab_version": (C.c_int, []),
    "ab_device_is_sm90": (C.c_int, []),
    "ab_generator_create": (C.c_int, [C.POINTER(GeneratorConfig), C.POINTER(_P)]),
    "ab_generator_destroy": (None, [_P]),
    "ab_generator_param_bytes": (C.c_size_t, [_P]),
    "ab_generator_bind_params": (C.c_int, [_P, _P, C.c_size_t]),
    "ab_generator_num_tensors": (C.c_int, [_P]),
    "ab_generator_tensor_name": (C.c_char_p, [_P, C.c_int]),
    "ab_generator_load_tensor": (C.c_int, [_P, C.c_char_p, _P, _I64P, C.c_int32, _P]),
    "ab_generator_load_weight_norm": (C.c_int, [_P, C.c_char_p, _P, _P, _I64P, C.c_int32, _P]),
    "ab_generator_finalize": (C.c_int, [_P, C.c_int32, _P]),
    "ab_generator_workspace_bytes": (C.c_size_t, [_P, C.c_int64, C.c_int64]),
    "ab_generator_forward": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _I64P, _P, _P, C.c_size_t, _P]),
    "ab_generator_forward_cond": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _I64P, _P, C.c_int64, _P, _P, C.c_size_t, _P]),
    "ab_generator_last_launches": (C.c_int, [_P]),
    "ab_generator_set_profiling": (C.c_int, [_P, C.c_int32]),
    "ab_generator_set_option": (C.c_int, [_P, C.c_char_p, C.c_int32]),
    "ab_generator_output_samples": (C.c_int64, [_P, C.c_int64, C.c_int64]),
    "ab_generator_set_tail_events": (C.c_int, [_P, C.POINTER(C.c_void_p), C.c_int32]),
    "ab_generator_get_profile": (C.c_int, [_P, C.POINTER(ProfileEntry), C.c_int32, C.POINTER(C.c_int32)]),
    "ab_diffwave_workspace_bytes": (C.c_size_t, [_P, C.c_int64, C.c_int64, C.c_int32]),
    "ab_diffwave_condition": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _I64P, C.POINTER(C.c_float), C.c_int32, _P,
                                        C.c_size_t, _P]),
    "ab_diffwave_step": (C.c_int, [_P, _P, C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_float, C.c_float, _P, _P, _P,
                                   C.c_size_t, _P]),
    "ab_diffwave_forward": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _P, _I64P, C.POINTER(C.c_float), C.c_int32, _P, _P,
                                      C.c_size_t, _P]),
    "ab_facodec_vq2emb": (C.c_int, [_P, _P, _I64P, C.c_int32, C.c_int64, C.c_int64, C.c_int32, _P, _P]),
    "ab_facodec_inference": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _I64P, _P, C.c_int64, _P, _P, C.c_size_t, _P]),
    "ab_facodec_quantize_workspace_bytes": (C.c_size_t, [_P, C.c_int64, C.c_int64]),
    "ab_facodec_quantize": (C.c_int, [_P, _P, _I64P, C.c_int64, C.c_int64, C.c_int32, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "ab_facodec_quantize_prosody": (C.c_int, [_P, _P, _I64P, _P, _I64P, C.c_int64, C.c_int64, C.c_int32, _P, _P, _P, _P,
                                              _P, C.c_size_t, _P]),
    "ab_facodec_prosody_input_forward": (C.c_int, [_P, _I64P, _P, _P, _P, C.c_int64, C.c_int64, _P, _P]),
    "ab_facodec_redecoder_vq2emb_workspace_bytes": (C.c_size_t, [_P, C.c_int64, C.c_int64]),
    "ab_facodec_redecoder_vq2emb": (C.c_int, [_P, _P, _I64P, C.c_int32, C.c_int64, C.c_int64, _P, C.c_int64, C.c_int32,
                                              _P, _P, C.c_size_t, _P]),
    "ab_rvq_quantize": (C.c_int, [_P, _P, _I64P, C.c_int64, C.c_int64, C.c_int32, _P, _P, _P, _P]),
    "ab_rvq_vq2emb": (C.c_int, [_P, _P, _I64P, C.c_int32, C.c_int64, C.c_int64, _P, _P]),
    "ab_facodec_encoder_frames": (C.c_int64, [_P, C.c_int64]),
    "ab_facodec_encode": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _I64P, _P, _P, C.c_size_t, _P]),
    "ab_activation1d_forward": (C.c_int, [_P, _P, C.c_int64, C.c_int64, C.c_int64, _P, _P, C.c_int32, _P, _P, _P]),
    "ab_activation1d_packed_forward": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int64, C.c_int64, _P, _P, C.c_int32,
                                                 C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int32, _P]),
    "ab_snake1d_forward": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int64, C.c_int64, _P, C.c_int32, _P]),
    "ab_conv1d_forward": (C.c_int, [_P, _P, _P, _P, _P, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int32,
                                    C.c_int32, C.c_float, C.c_int32, C.c_int32, _P, C.c_size_t, _P]),
    "ab_conv1d_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int32, C.c_int32]),
    "ab_conv_transpose1d_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32]),
    "ab_conv_transpose1d_forward": (C.c_int, [_P, _P, _P, _P, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                              C.c_int32, C.c_int32, C.c_float, C.c_int32, _P, C.c_size_t, _P]),
    "ab_tc_conv_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int64, C.c_int64, C.c_int32, C.c_int32]),
    "ab_tc_conv_forward": (C.c_int, [C.c_int32, _P, _I64P, C.c_float, _P, _P, _P, _P, _P, C.c_float, C.c_int32, _P, _P,
                                     C.c_float, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                     C.c_int32, _P, C.c_size_t, _P]),
    "ab_vocos_norm_forward": (C.c_int, [_P, _P, _P, _P, _P, C.c_float, _P, _P, C.c_int32, C.c_int64, C.c_int64,
                                        C.c_int64, _P]),
    "ab_vocos_pointwise_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                                        C.c_int32]),
    "ab_vocos_pointwise_forward": (C.c_int, [C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int64, C.c_int64,
                                             C.c_int64, C.c_int64, C.c_int32, _P, C.c_size_t, _P]),
    "ab_diffwave_layer_workspace_bytes": (C.c_size_t, [C.c_int32]),
    "ab_diffwave_layer_forward": (C.c_int, [_P, _P, C.c_int64, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int64, C.c_int64,
                                            C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, C.c_size_t, _P]),
    "ab_diffwave_tail_forward": (C.c_int, [_P, _P, _P, _P, _P, C.c_float, C.c_int64, C.c_int64, _P, _P, _P, C.c_float,
                                           C.c_float, C.c_float, _P]),
    "ab_diffwave_upsample_forward": (C.c_int, [_P, _I64P, _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int64, C.c_int32,
                                               C.c_int64, _P, _P]),
    "ab_mel_create": (C.c_int, [C.POINTER(MelConfig), C.POINTER(_P)]),
    "ab_mel_destroy": (None, [_P]),
    "ab_mel_num_frames": (C.c_int64, [_P, C.c_int64]),
    "ab_mel_workspace_bytes": (C.c_size_t, [_P, C.c_int64, C.c_int64]),
    "ab_mel_forward": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _P, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "ab_mel_forward_fused": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "ab_mel_backward_workspace_bytes": (C.c_size_t, [_P, C.c_int64, C.c_int64]),
    "ab_mel_backward": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "ab_amplitude_phase_forward": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _P, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "ab_spectral_head_forward": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int64, C.c_int64, C.c_float, _P, _P, _P, _P, _P]),
    "ab_istft_workspace_bytes": (C.c_size_t, [_P, C.c_int64, C.c_int64]),
    "ab_istft_forward": (C.c_int, [_P, _P, C.c_int64, C.c_int64, _P, _P, _P, C.c_size_t, _P]),
    "ab_pcm16_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "ab_pcm16_forward": (C.c_int, [_P, C.c_int64, C.c_int64, C.c_int64, _P, C.c_int32, C.c_float, C.c_int64, _P, C.c_int64,
                                   _P, C.c_size_t, _P]),
}


def _load() -> C.CDLL:
    path = _build.LIB
    if _build.needs_build():
        try:
            _build.build()
        except Exception as e:  # no nvcc on this machine: use the shipped binary if there is one
            if not os.path.exists(path):
                raise RuntimeError(
                    "amphion_b200: libamphion_b200.so is missing and could not be built "
                    f"({e}). Run `python -m amphion_b200.build` on a machine with nvcc. "
                    "There is no CPU fallback.") from e
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()
LIB_PATH = _build.LIB


def last_error() -> str:
    return (lib.ab_last_error() or b"").decode()


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"amphion_b200: {what} failed (code {rc}): {last_error()}")


def shape_array(shape):
    return (C.c_int64 * len(shape))(*[int(s) for s in shape])


def require_cuda(t, what: str):
    if not t.is_cuda:
        raise RuntimeError(
            f"amphion_b200: {what} needs a CUDA tensor (got device '{t.device}'); there is no CPU fallback")
    return t


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())
