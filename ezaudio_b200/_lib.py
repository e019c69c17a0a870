"""ctypes binding of libezb200.so (include/ezb200.h).  No fallback: a missing library raises."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libezb200.so")


class EzbError(RuntimeError):
    pass


class DitDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("embed_dim", "num_heads", "depth", "context_dim", "inner_dim", "ada_rank")] + \
               [("ada_scaling", C.c_float)] + \
               [(n, C.c_int32) for n in ("latent_chans", "is_controlnet", "cond_c0", "cond_c1", "max_batch", "max_len",
                                         "max_ctx_len", "max_timesteps", "precision")]


class VaeDesc(C.Structure):
    _fields_ = [("latent_dim", C.c_int32), ("channels", C.c_int32), ("out_channels", C.c_int32), ("n_stages", C.c_int32),
                ("c_mults", C.c_int32 * 8), ("strides", C.c_int32 * 8), ("max_batch", C.c_int32),
                ("max_latent_len", C.c_int32), ("precision", C.c_int32), ("with_encoder", C.c_int32), ("in_channels", C.c_int32),
                ("enc_latent_dim", C.c_int32)]


class T5Desc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("vocab_size", "d_model", "d_kv", "num_heads", "d_ff", "num_layers", "num_buckets", "max_distance")] + \
               [("eps", C.c_float)] + [(n, C.c_int32) for n in ("max_batch", "max_len", "precision")]


class DdimSlot(C.Structure):
    """ezb_ddim_slot: the CFG / DDIM constants of one sample of ezb_cfg_ddim_step_slots."""
    _fields_ = [("guidance_scale", C.c_float), ("guidance_rescale", C.c_float), ("coef", C.c_float * 5), ("flags", C.c_int32)]


class DpmSlot(C.Structure):
    """ezb_dpm_slot: the CFG / DPM-Solver++ constants of one sample of ezb_cfg_dpm_step_slots."""
    _fields_ = [("guidance_scale", C.c_float), ("guidance_rescale", C.c_float), ("coef", C.c_float * 7), ("flags", C.c_int32)]


SLOT_ACTIVE, SLOT_CFG, SLOT_ORDER2 = 1, 2, 4   # ezb_ddim_slot.flags / ezb_dpm_slot.flags


class TestEpilogue(C.Structure):
    _fields_ = [("bias", C.c_void_p), ("bias_mod", C.c_int32), ("resid", C.c_void_p), ("ldr", C.c_int32),
                ("gate", C.c_void_p), ("gate_bstride", C.c_int32), ("rows_per_batch", C.c_int32),
                ("out_f32", C.c_void_p), ("ld32", C.c_int32), ("out_bf16", C.c_void_p), ("ld16", C.c_int32),
                ("split_stride", C.c_int32), ("act", C.c_int32), ("act_a", C.c_void_p), ("act_b", C.c_void_p),
                ("fin_st", C.c_void_p), ("fin_slots", C.c_int32), ("fin_ld_st", C.c_int32), ("fin_inv_dim", C.c_float), ("fin_u", C.c_void_p),
                ("fin_v", C.c_void_p), ("fout_st", C.c_void_p), ("fout_ld_st", C.c_int32), ("fout_a0", C.c_void_p), ("fout_ld0", C.c_int32),
                ("fout_g0", C.c_void_p), ("fout_a1", C.c_void_p), ("fout_ld1", C.c_int32), ("fout_g1", C.c_void_p),
                ("fin_st1", C.c_void_p), ("fin_slots1", C.c_int32)]


class TestHeadsArgs(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("B", "L", "D", "H", "dh", "nsec")] + [("kinds", C.c_int32 * 3)] + \
               [(n, C.c_void_p) for n in ("norm_q", "norm_k", "inv_freq")] + [("rope", C.c_int32)] + \
               [(n, C.c_void_p) for n in ("q", "k", "vt")] + [(n, C.c_int32) for n in ("ld_qk", "dvp", "Lpad")] + \
               [("fold_st", C.c_void_p), ("fold_slots", C.c_int32), ("fold_ld_st", C.c_int32), ("fold_u", C.c_void_p),
                ("fold_v", C.c_void_p), ("variant", C.c_int32)]


class TestLinearArgs(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("M", "N", "K", "kmul", "lda")] + [(n, C.c_void_p) for n in ("A", "W", "w_packed", "bias", "resid")] + \
               [("ldr", C.c_int32), ("gate", C.c_void_p)] + [(n, C.c_int32) for n in ("gate_bstride", "rows_per_batch")] + \
               [("out_f32", C.c_void_p), ("ld32", C.c_int32), ("out_bf16", C.c_void_p)] + [(n, C.c_int32) for n in ("ld16", "split", "act")] + \
               [("out_scale", C.c_float), ("scale", C.c_void_p)] + [(n, C.c_int32) for n in ("kernel", "pair", "swap_ab", "m_select")] + \
               [("ran", C.POINTER(C.c_int32))]


class TestVaeArgs(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("kind", "precision", "B", "T", "cin", "cout", "taps", "dil", "stride")] + \
               [(n, C.c_void_p) for n in ("weight_v", "weight_g", "bias", "alpha", "beta", "x", "resid", "noise", "raw", "act", "out",
                                          "w_packed")]


class TestFp8Args(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("kind", "M", "D")] + \
               [(n, C.c_void_p) for n in ("x", "weight", "bias", "shift", "scale", "q", "s")] + [("inner", C.c_int32)] + \
               [(n, C.c_void_p) for n in ("w", "b", "out")] + [(n, C.c_int32) for n in ("B", "L", "H", "dh")] + \
               [(n, C.c_void_p) for n in ("norm_q", "norm_k", "inv_freq")] + [("rope", C.c_int32)] + \
               [(n, C.c_void_p) for n in ("q_out", "k_out", "vt_out")] + [(n, C.c_int32) for n in ("ld_qk", "dvp", "Lpad")] + \
               [(n, C.c_void_p) for n in ("w_q", "w_s")]


class TestStepArgs(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("kind", "variant", "M", "D1", "D2", "kmul", "mod_bstride", "rows_per_batch", "B", "L", "C", "Kp",
                                         "H", "dh", "nsec", "in_bf16")] + \
               [("kinds", C.c_int32 * 3), ("col_off", C.c_int32 * 3)] + \
               [(n, C.c_int32) for n in ("ld_in", "ld_qk", "Lpad", "dv_pad", "R", "N", "K", "ld_add", "ld_out", "act")] + \
               [("out_scale", C.c_float)] + \
               [(n, C.c_void_p) for n in ("x", "x2", "x3", "w", "b", "shift", "scale", "G", "Cc", "gt", "gt_mask", "mask_embed", "add", "lens",
                                          "norm_q", "norm_k", "inv_freq", "out")] + \
               [("f32_out", C.c_void_p * 3), ("bf_out", C.c_void_p * 3)]


class TestFoldArgs(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("kind", "variant", "M", "N", "K", "R", "inner", "geglu_bn", "bn")] + \
               [(n, C.c_void_p) for n in ("w", "b", "shift", "scale")] + [(n, C.c_int32) for n in ("ld_mod", "rows_per_batch")] + \
               [(n, C.c_void_p) for n in ("W", "bias", "add_v", "w_packed", "G", "Cc", "u", "v", "A", "st")] + \
               [(n, C.c_int32) for n in ("slots", "ld_st")] + \
               [(n, C.c_void_p) for n in ("out", "W2", "b2", "x", "gate")] + [("gate_bstride", C.c_int32)] + \
               [(n, C.c_void_p) for n in ("fout_st", "a0", "g0", "grid_barrier", "W16", "resid", "out_f32", "x2", "x3")] + \
               [("D2", C.c_int32), ("ln_out", C.c_void_p), ("ran_bn", C.c_int32), ("ran_fused", C.c_int32)]


class TestCondArgs(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("kind", "M", "D", "F", "kmul", "vocab")] + [("eps", C.c_float)] + \
               [(n, C.c_int32) for n in ("B", "L", "H", "dk", "c0", "c1", "stage")] + \
               [(n, C.c_void_p) for n in ("in_", "w", "b", "k", "v", "key_mask", "out", "out32", "out_v")]


_lib = None

_VP, _I, _F = C.c_void_p, C.c_int, C.c_float
_SIGS = {
    "ezb_version": ([], C.c_int),
    "ezb_last_error": ([], C.c_char_p),
    "ezb_dit_create": ([C.POINTER(_VP), C.POINTER(DitDesc), _I], _I),
    "ezb_dit_destroy": ([_VP], _I),
    "ezb_dit_load_weight": ([_VP, C.c_char_p, _VP, C.POINTER(C.c_int64), _I, _VP], _I),
    "ezb_dit_finalize_weights": ([_VP, _VP], _I),
    "ezb_dit_set_context": ([_VP, _VP, _VP, _I, _I, _VP], _I),
    "ezb_dit_set_timesteps": ([_VP, C.POINTER(C.c_int64), _I, _VP], _I),
    "ezb_dit_forward": ([_VP, _VP, _VP, _VP, C.POINTER(C.c_int32), _I, C.POINTER(_VP), _VP, _I, _I, _VP, _VP], _I),
    "ezb_controlnet_forward": ([_VP, _VP, _VP, _VP, C.POINTER(C.c_int32), _I, _VP, _F, C.POINTER(_VP), _I, _I, _VP], _I),
    "ezb_cfg_ddim_step": ([_I, _VP, _VP, _VP, _I, _I, _I, _F, _F, C.POINTER(C.c_float), _VP, _VP], _I),
    "ezb_dit_set_context_rows": ([_VP, _VP, _VP, _I, _I, _I, _VP], _I),
    "ezb_dit_forward_tdev": ([_VP, _VP, _VP, _VP, _VP, C.POINTER(_VP), _VP, _I, _I, _VP, _VP], _I),
    "ezb_cfg_ddim_step_slots": ([_I, _VP, _VP, _VP, _VP, _I, _I, _I, _VP, _VP], _I),
    "ezb_cfg_dpm_step": ([_I, _VP, _VP, _VP, _VP, _I, _I, _I, _F, _F, C.POINTER(C.c_float), _I, _VP, _VP], _I),
    "ezb_cfg_dpm_step_slots": ([_I, _VP, _VP, _VP, _VP, _VP, _I, _I, _I, _VP, _VP], _I),
    "ezb_window_gather": ([_I, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _VP], _I),
    "ezb_window_blend": ([_I, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _VP], _I),
    "ezb_loop_gather": ([_I, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _VP], _I),
    "ezb_loop_blend": ([_I, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _VP], _I),
    "ezb_timeline_gather": ([_I, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _VP], _I),
    "ezb_timeline_guide": ([_I, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _F, _F, _VP], _I),
    "ezb_timeline_blend": ([_I, _VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _VP], _I),
    "ezb_controlnet_set_condition": ([_VP, _VP, _I, _I, _VP], _I),
    "ezb_controlnet_set_condition_rows": ([_VP, _VP, _I, _I, _I, _VP], _I),
    "ezb_controlnet_forward_tdev": ([_VP, _VP, _VP, _VP, C.POINTER(_VP), _I, _I, _VP], _I),
    "ezb_controlnet_forward_cached": ([_VP, _VP, _VP, _VP, C.POINTER(C.c_int32), _I, _F, C.POINTER(_VP), _I, _I, _VP], _I),
    "ezb_option_epoch": ([], C.c_ulonglong),
    "ezb_vae_create": ([C.POINTER(_VP), C.POINTER(VaeDesc), _I], _I),
    "ezb_vae_destroy": ([_VP], _I),
    "ezb_vae_load_weight": ([_VP, C.c_char_p, _VP, C.POINTER(C.c_int64), _I, _VP], _I),
    "ezb_vae_finalize_weights": ([_VP, _VP], _I),
    "ezb_vae_decode": ([_VP, _VP, _VP, _I, _I, _VP], _I),
    "ezb_vae_encode": ([_VP, _VP, _VP, _VP, _I, _I, _VP], _I),
    "ezb_vae_decode_lens": ([_VP, _VP, _VP, _I, _I, _VP, _VP], _I),
    "ezb_vae_encode_lens": ([_VP, _VP, _VP, _VP, _I, _I, _VP, _VP], _I),
    "ezb_vae_encode_noised": ([_VP, _VP, _VP, _VP, _VP, _F, _F, _VP, _I, _I, _VP, _VP], _I),
    "ezb_t5_create": ([C.POINTER(_VP), C.POINTER(T5Desc), _I], _I),
    "ezb_t5_destroy": ([_VP], _I),
    "ezb_t5_load_weight": ([_VP, C.c_char_p, _VP, C.POINTER(C.c_int64), _I, _VP], _I),
    "ezb_t5_finalize_weights": ([_VP, _VP], _I),
    "ezb_t5_forward": ([_VP, _VP, _VP, _VP, _VP, _I, _I, _VP], _I),
    "ezb_energy_condition": ([_I, _VP, _VP, _I, _I, _I, _I, _F, _I, _I, _VP], _I),
    "ezb_wave_prepare": ([_I, _VP, _VP, _I, _I, _I, _I, _F, _VP], _I),
    "ezb_wave_splice": ([_I, _VP, C.c_longlong, _VP, C.c_longlong, C.c_longlong, _VP], _I),
    "ezb_wave_to_pcm16": ([_I, _VP, _VP, C.c_longlong, _VP], _I),
    "ezb_set_option": ([C.c_char_p, _I], _I),
    "ezb_debug_read": ([C.POINTER(C.c_ulonglong)], _I),
    "ezb_launch_count": ([], C.c_ulonglong),
    "ezb_launch_count_add": ([C.c_ulonglong], None),
    "ezb_ln_launch_count": ([_I], C.c_ulonglong),
    "ezb_attn_launch_count": ([_I], C.c_ulonglong),
    "ezb_prof_gemm_begin": ([], _I),
    "ezb_prof_gemm_end": ([C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_double)], _I),
    "ezb_prof_gemm_stats": ([C.c_double, C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_double)], _I),
    "ezb_test_gemm": ([_I, _VP, _I, _VP, _I, _I, _I, _I, _I, _I, C.POINTER(TestEpilogue), _I, _I, _I, _I, _I, _I, _VP], _I),
    "ezb_test_attention": ([_I, _VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _VP], _I),
    "ezb_test_attention_lens": ([_I, _VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _VP], _I),
    "ezb_test_heads": ([_I, _VP, _VP, C.POINTER(TestHeadsArgs), _VP], _I),
    "ezb_test_mlp": ([_I, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _I, _I, _VP, _VP, _I, _I, _I, _I, _VP], _I),
    "ezb_test_linear": ([_I, C.POINTER(TestLinearArgs), _VP], _I),
    "ezb_test_vae": ([_I, C.POINTER(TestVaeArgs), _VP], _I),
    "ezb_test_fp8": ([_I, C.POINTER(TestFp8Args), _VP], _I),
    "ezb_test_step": ([_I, C.POINTER(TestStepArgs), _VP], _I),
    "ezb_test_cond": ([_I, C.POINTER(TestCondArgs), _VP], _I),
    "ezb_test_fold": ([_I, C.POINTER(TestFoldArgs), _VP], _I),
}
EXPORTS = tuple(_SIGS)


def lib():
    """Loads the library (once).  Raises EzbError when it has not been built -- there is no CPU path."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EzbError(f"{LIB_PATH} not found: run `python -m ezaudio_b200.build` (or __graft_entry__.build()); "
                           "ezaudio_b200 has no CPU / PyTorch fallback")
        L = C.CDLL(LIB_PATH)
        for name, (args, res) in _SIGS.items():
            fn = getattr(L, name)  # AttributeError if the symbol is missing
            fn.argtypes, fn.restype = args, res
        _lib = L
    return _lib


def check(rc: int):
    if rc != 0:
        raise EzbError(f"libezb200 error {rc}: {lib().ezb_last_error().decode()}")


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
