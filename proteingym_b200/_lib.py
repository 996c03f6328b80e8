"""ctypes binding of libpgscore.so (include/pgscore.h). There is no CPU fallback: if the library is missing or there
is no sm_90 device, calls fail loudly."""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpgscore.so")

PG_ARCH_ESM1B, PG_ARCH_ESM2, PG_ARCH_TRANCEPTION, PG_ARCH_MSA, PG_ARCH_ESMC, PG_ARCH_RITA, PG_ARCH_PROGEN2 = 0, 1, 2, 3, 4, 5, 6
PG_ARCH_PROTGPT2 = 7
PG_ARCH_POET = 8
PG_ARCH_PROGEN3 = 9
PG_PREC_F16, PG_PREC_F16X3, PG_PREC_F16F8, PG_PREC_F16D = 0, 1, 2, 3
PRECISIONS = {"f16": PG_PREC_F16, "f16x3": PG_PREC_F16X3, "f16f8": PG_PREC_F16F8, "f16d": PG_PREC_F16D}


class PgModelDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("arch", "layers", "embed_dim", "heads", "ffn_dim", "vocab", "max_positions",
                                         "token_dropout", "emb_ln_before", "precision", "device", "max_rows",
                                         "kv_heads", "n_experts", "top_k", "gated_mlp")] + [("rms_eps", C.c_float)]


class PgTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("shape", C.c_int64 * 2)]


class PgGemmArgs(C.Structure):
    _fields_ = [("a", C.c_void_p), ("lda", C.c_int64), ("w", C.c_void_p), ("ldw", C.c_int64), ("bias", C.c_void_p),
                ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("nseg", C.c_int32), ("epi", C.c_int32),
                ("out_h", C.c_void_p), ("ldo", C.c_int64), ("out_lo_off", C.c_int64),
                ("resid", C.c_void_p), ("ldr", C.c_int64),
                ("rot_cos", C.c_void_p), ("rot_sin", C.c_void_p), ("rot_T", C.c_int32), ("rot_dim", C.c_int32),
                ("a_scale", C.c_float), ("w_inv", C.c_void_p), ("out_fmt", C.c_int32), ("out_scale", C.c_float),
                ("grp_rows_a", C.c_int32), ("grp_rows_b", C.c_int32),
                ("base_pre", C.c_void_p), ("base_post", C.c_void_p), ("base_T", C.c_int32), ("mask_pos", C.c_void_p)]


class PgAttnArgs(C.Structure):
    _fields_ = [("qkv", C.c_void_p), ("ld", C.c_int64), ("lo_off", C.c_int64),
                ("out", C.c_void_p), ("ldo", C.c_int64), ("out_lo_off", C.c_int64),
                ("B", C.c_int32), ("T", C.c_int32), ("heads", C.c_int32), ("nseg", C.c_int32),
                ("causal", C.c_int32), ("alibi_slopes", C.c_void_p), ("impl", C.c_int32),
                ("out_fmt", C.c_int32), ("out_scale", C.c_float),
                ("base_o", C.c_void_p), ("mask_pos", C.c_void_p), ("cout", C.c_void_p), ("ldc", C.c_int64), ("c_lo_off", C.c_int64)]


class PgAttnForm(C.Structure):
    _fields_ = [("prefix", C.c_void_p), ("prefix_len", C.c_int32), ("prefix_mem", C.c_int32), ("seg_start", C.c_void_p),
                ("perm_C", C.c_int32), ("head_dim", C.c_int32)]


class PgGemmForm(C.Structure):
    _fields_ = [("rot_pos", C.c_void_p), ("rot_half", C.c_int32), ("kchunk", C.c_int32), ("w_uniform", C.c_int32),
                ("lm_part", C.c_void_p), ("lm_tgt", C.c_void_p), ("lm_logits", C.c_void_p), ("lm_ids", C.c_void_p),
                ("lm_lens", C.c_void_p), ("lm_T", C.c_int32), ("rg_expert", C.c_void_p), ("rg_tiles", C.c_void_p),
                ("rg_pad", C.c_int32), ("rg_experts", C.c_int32)]


class PgArFusion(C.Structure):
    _fields_ = [("log_prior", C.c_void_p), ("prior_row", C.c_void_p), ("alpha", C.c_float),
                ("log_prior2", C.c_void_p), ("prior_row2", C.c_void_p), ("beta", C.c_float),
                ("first_col", C.c_int32), ("out_logprobs", C.c_void_p)]


class PgLnForm(C.Structure):
    _fields_ = [("dp", C.c_int32), ("perm_R", C.c_int32), ("perm_C", C.c_int32), ("base", C.c_void_p), ("base_T", C.c_int32)]


class PgEsmEmbedArgs(C.Structure):
    _fields_ = [("tokens", C.c_void_p), ("n_tokens", C.c_int32), ("positions", C.c_void_p), ("win_start", C.c_void_p),
                ("P", C.c_int32), ("T", C.c_int32), ("d", C.c_int32), ("embed", C.c_void_p), ("pos_table", C.c_void_p),
                ("lnb_gamma", C.c_void_p), ("lnb_beta", C.c_void_p), ("token_dropout", C.c_int32), ("mask_idx", C.c_int32),
                ("p_offset", C.c_int32), ("force_mask_scale", C.c_int32), ("x", C.c_void_p)]


class PgMlmHeadArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("d", C.c_int32), ("T", C.c_int32), ("row_in_seq", C.c_void_p), ("P", C.c_int32),
                ("all_rows", C.c_int32)] + [(n, C.c_void_p) for n in ("lna_g", "lna_b", "dense_w", "dense_b", "ln_g", "ln_b",
                                                                      "out_w", "out_b")] + \
        [("vocab", C.c_int32), ("scratch_a", C.c_void_p), ("scratch_b", C.c_void_p), ("out", C.c_void_p)]


class PgArHeadArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("d", C.c_int32), ("B", C.c_int32), ("T", C.c_int32), ("vocab", C.c_int32),
                ("ids", C.c_void_p), ("lens", C.c_void_p), ("lnf_g", C.c_void_p), ("lnf_b", C.c_void_p),
                ("wte", C.c_void_p), ("bias", C.c_void_p), ("label_off", C.c_int32), ("ignore_id", C.c_int32),
                ("tok_logp", C.c_void_p), ("out_sum", C.c_void_p)]


# every symbol include/pgscore.h declares, with its ctypes signature
SIGNATURES = {
    "pg_abi_version": (C.c_int, []),
    "pg_create": (C.c_int, [C.POINTER(PgModelDesc), C.POINTER(C.c_void_p)]),
    "pg_load_weights": (C.c_int, [C.c_void_p, C.POINTER(PgTensor), C.c_int32]),
    "pg_destroy": (C.c_int, [C.c_void_p]),
    "pg_last_error": (C.c_char_p, [C.c_void_p]),
    "pg_masked_marginals": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                      C.c_int32, C.c_void_p, C.c_void_p]),
    "pg_msa_masked_marginals": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_void_p]),
    "pg_forward_logprobs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_void_p]),
    "pg_score_mutants": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_int32, C.c_void_p, C.c_void_p]),
    "pg_ar_loglik": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p,
                               C.c_void_p]),
    "pg_ar_loglik_fused": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(PgArFusion), C.c_void_p,
                                     C.c_void_p]),
    "pg_ar_prefix_begin": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(PgArFusion), C.c_void_p, C.c_void_p]),
    "pg_ar_loglik_prefix": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(PgArFusion),
                                      C.c_void_p, C.c_void_p]),
    "pg_poet_context": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_void_p]),
    "pg_poet_loglik": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_poet_record": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]),
    "pg_gemm": (C.c_int, [C.POINTER(PgGemmArgs), C.c_void_p]),
    "pg_gemm_form": (C.c_int, [C.POINTER(PgGemmArgs), C.POINTER(PgGemmForm), C.c_void_p]),
    "pg_layernorm_f16": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                   C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_void_p]),
    "pg_layernorm_form": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                    C.c_int64, C.c_int64, C.c_int32, C.c_float, C.POINTER(PgLnForm), C.c_void_p]),
    "pg_pack_weight": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_attention": (C.c_int, [C.POINTER(PgAttnArgs), C.c_void_p]),
    "pg_attention_form": (C.c_int, [C.POINTER(PgAttnArgs), C.POINTER(PgAttnForm), C.c_void_p]),
    "pg_attention_rows": (C.c_int, [C.POINTER(PgAttnArgs), C.c_void_p, C.c_void_p]),
    "pg_qk_ln_rotary": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_int32, C.c_void_p]),
    "pg_esm_embed": (C.c_int, [C.POINTER(PgEsmEmbedArgs), C.c_void_p]),
    "pg_mlm_head": (C.c_int, [C.POINTER(PgMlmHeadArgs), C.c_void_p]),
    "pg_ar_head": (C.c_int, [C.POINTER(PgArHeadArgs), C.POINTER(PgArFusion), C.c_void_p]),
    "pg_lm_combine": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_msa_cluster_neighbors": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pg_msa_prior": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_void_p, C.c_void_p]),
    "pg_eve_output_conv": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "pg_progen3_routing": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p]),
    "pg_set_tuning": (C.c_int, [C.c_char_p, C.c_int32]),
    "pg_launch_count": (C.c_longlong, []),
    "pg_profile_begin": (C.c_int, []),
    "pg_profile_end": (C.c_int, [C.POINTER(C.c_float), C.POINTER(C.c_int32), C.c_int32]),
}

PROFILE_CATEGORIES = ["embed", "layernorm", "gemm_qkv", "attention", "gemm_out", "gemm_fc1", "gemm_fc2", "head", "score",
                      "other", "tied_gemm", "regroup"]

_lib = None


class PgError(RuntimeError):
    pass


def load():
    """Load the shared library (building it is ``__graft_entry__.build()`` / ``python -m proteingym_b200.build``)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PgError(f"{LIB_PATH} is missing: run `python -m proteingym_b200.build` (nvcc, sm_90a). "
                          "There is no CPU/PyTorch fallback for the scoring path.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc: int, handle=None):
    if rc != 0:
        msg = load().pg_last_error(handle)
        raise PgError(f"libpgscore error {rc}: {msg.decode() if msg else '?'}")


class Model:
    """Owner of one libpgscore handle: ``pg_create`` from a PgModelDesc, then ``pg_load_weights`` from fp32 tensors staged on the device
    (the library repacks them; the staging copy is freed before the constructor returns). ``close()`` (also on garbage collection)
    destroys the handle; it is safe on an object whose constructor never ran."""
    handle = None

    def __init__(self, desc: PgModelDesc, tensors: dict, device: int = 0):
        if not torch.cuda.is_available():
            raise PgError("no CUDA device: the H100 scorer has no CPU fallback")
        self.lib = load()
        self.device = torch.device("cuda", device)
        self.handle = C.c_void_p()
        check(self.lib.pg_create(C.byref(desc), C.byref(self.handle)))
        try:
            gpu = [(n, t.to(self.device, torch.float32).contiguous()) for n, t in tensors.items()]
            arr = (PgTensor * len(gpu))()
            for i, (n, t) in enumerate(gpu):
                arr[i].name = n.encode()
                arr[i].data = t.data_ptr()
                arr[i].shape[0] = t.shape[0]
                arr[i].shape[1] = t.shape[1] if t.dim() == 2 else 1
            torch.cuda.synchronize(self.device)
            check(self.lib.pg_load_weights(self.handle, arr, len(gpu)), self.handle)
            del gpu
            torch.cuda.empty_cache()
        except Exception:
            self.close()
            raise

    def stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def close(self):
        if self.handle:
            self.lib.pg_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
