"""ctypes binding of libsgformer_b200.so (the C-ABI declared in include/sgformer_b200.h).

The library is built in-tree by `sgformer_b200._build.build()` / `__graft_entry__.build()`.  There is no fallback:
if the library is missing, or a launch fails, a RuntimeError is raised."""
import ctypes as C
import os

from . import _build

_i32, _i64, _f32, _u64, _vp, _sz = C.c_int32, C.c_int64, C.c_float, C.c_uint64, C.c_void_p, C.c_size_t
SGF_MAX_SRC, SGF_MAX_SEG = 4, 16
F32, BF16 = 0, 1
EPI_AFFINE, EPI_ATTN_APPLY, EPI_ATTN_GRAM = 0, 1, 2


class GemmNtArgs(C.Structure):
    _fields_ = [
        ("a", _vp * SGF_MAX_SRC), ("lda", _i64 * SGF_MAX_SRC), ("a_cols", _i64 * SGF_MAX_SRC),
        ("b", _vp * SGF_MAX_SRC), ("ldb", _i64 * SGF_MAX_SRC), ("b_cols", _i64 * SGF_MAX_SRC),
        ("n_a", _i32), ("n_b", _i32), ("n_seg", _i32),
        ("seg_a", _i32 * SGF_MAX_SEG), ("seg_akoff", _i32 * SGF_MAX_SEG), ("seg_b", _i32 * SGF_MAX_SEG),
        ("seg_bkoff", _i32 * SGF_MAX_SEG), ("seg_klen", _i32 * SGF_MAX_SEG),
        ("b_tail", _vp), ("ldb_tail", _i64),
        ("rows", _i64), ("n_out", _i32),
        ("epi", _i32),
        ("out", _vp), ("ldo", _i64), ("out_dtype", _i32),
        ("bias", _vp),
        ("aux", _vp), ("ld_aux", _i64), ("aux_dtype", _i32),
        ("row_scale", _vp),
        ("alpha", _f32), ("beta", _f32),
        ("alpha_dev", _vp), ("beta_dev", _vp),
        ("relu", _i32), ("accumulate", _i32),
        ("nf", _f32), ("nf_dev", _vp),
        ("den_out", _vp),
        ("r1_row", _vp), ("r1_col", _vp),
        ("col_sum", _vp), ("col_sumsq", _vp),
        ("schedule", _i32),
    ]


class AttnGramArgs(C.Structure):
    """sgf_attn_gram_args (include/sgformer_b200.h): every pointer is device fp32."""
    _fields_ = [
        ("h", _i32), ("m", _i32), ("d", _i32), ("n_nodes", _i64),
        ("wq", _vp), ("bq", _vp), ("wk", _vp), ("bk", _vp), ("wv", _vp), ("bv", _vp),
        ("ld_wq", _i64), ("ld_wk", _i64), ("ld_wv", _i64),
        ("G", _vp), ("s", _vp),
        ("kx", _vp), ("qx", _vp), ("vx", _vp), ("z1", _vp), ("q1", _vp), ("v1", _vp), ("S", _vp),
        ("Bt", _vp), ("tail", _vp), ("bt", _vp), ("sc", _vp),
        # backward
        ("P", _vp), ("pg", _vp), ("cs", _vp), ("sg", _vp),
        ("dwq", _vp), ("dbq", _vp), ("dwk", _vp), ("dbk", _vp), ("dwv", _vp), ("dbv", _vp),
        ("bcat", _vp), ("a4", _vp),
        ("ws", _vp), ("ws_floats", _i64),
    ]


SGF_ADAM_MAX_TENSORS = 32


class AdamArgs(C.Structure):
    _fields_ = [
        ("n_tensors", _i32),
        ("param", _vp * SGF_ADAM_MAX_TENSORS), ("grad", _vp * SGF_ADAM_MAX_TENSORS),
        ("exp_avg", _vp * SGF_ADAM_MAX_TENSORS), ("exp_avg_sq", _vp * SGF_ADAM_MAX_TENSORS),
        ("numel", _i64 * SGF_ADAM_MAX_TENSORS),
        ("lr", _f32 * SGF_ADAM_MAX_TENSORS), ("beta1", _f32 * SGF_ADAM_MAX_TENSORS), ("beta2", _f32 * SGF_ADAM_MAX_TENSORS),
        ("eps", _f32 * SGF_ADAM_MAX_TENSORS), ("weight_decay", _f32 * SGF_ADAM_MAX_TENSORS),
        ("step", _vp * SGF_ADAM_MAX_TENSORS),
        ("chunk0", _i32 * (SGF_ADAM_MAX_TENSORS + 1)),
    ]


class GemmTnArgs(C.Structure):
    _fields_ = [
        ("a", _vp), ("lda", _i64), ("m", _i32),
        ("b", _vp), ("ldb", _i64), ("n", _i32),
        ("rows", _i64),
        ("out", _vp), ("ldo", _i64), ("transpose_out", _i32),
        ("alpha", _f32), ("beta", _f32), ("alpha_dev", _vp),
        ("ws", _vp), ("ws_bytes", _sz),
        ("n_pairs", _i32), ("a_off", _i32 * 6), ("b_off", _i32 * 6),
    ]


_SIGS = {
    "sgf_version": (C.c_char_p, []),
    "sgf_launch_count": (_i64, []),
    "sgf_set_device": (C.c_int, [C.c_int]),
    "sgf_csr_build_ws_bytes": (C.c_int, [_i64, _i64, C.POINTER(_sz)]),
    "sgf_csr_build": (C.c_int, [_vp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sgf_csr_build_rect": (C.c_int, [_vp, _i64, _i64, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sgf_subgraph_ws_bytes": (C.c_int, [_i64, _i64, C.POINTER(_sz)]),
    "sgf_to_undirected_ws_bytes": (C.c_int, [_i64, _i64, C.POINTER(_sz)]),
    "sgf_edge_symmetry": (C.c_int, [_vp, _i64, _i64, _vp, _vp]),
    "sgf_to_undirected": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _sz, _vp]),
    "sgf_remove_self_loops_ws_bytes": (C.c_int, [_i64, C.POINTER(_sz)]),
    "sgf_remove_self_loops": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _sz, _vp]),
    "sgf_add_self_loops": (C.c_int, [_vp, _i64, _i64, _vp, _vp]),
    "sgf_subgraph": (C.c_int, [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sgf_spmm": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _i64, _i64, C.c_int, C.c_int, _i64, _vp]),
    "sgf_spmm_flagged": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _i64, _i64, C.c_int, C.c_int, _i64, _vp, _i64, C.c_int, _vp]),
    "sgf_spmm_range": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _i64, _vp]),
    "sgf_csr_row_splits": (C.c_int, [_vp, _vp, _i64, _vp, C.c_int, _vp, _vp]),
    "sgf_signal": (C.c_int, [_vp, C.c_uint32, _vp]),
    "sgf_set_dropout_epoch": (C.c_int, [_vp]),
    "sgf_advance_dropout_epoch": (C.c_int, [_vp, _vp]),
    "sgf_memcpy_async": (C.c_int, [_vp, _vp, _sz, _vp]),
    "sgf_wait_flags": (C.c_int, [_vp, C.c_int, _vp]),
    "sgf_csr_build_rot": (C.c_int, [_vp, _i64, _i64, _i64, _i64, C.c_int, C.c_int, _i64, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sgf_spmm_heavy": (C.c_int, [_vp, _vp, _vp, _i64, _vp, _i64, C.c_int, C.c_int, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _vp]),
    "sgf_gemm_nt": (C.c_int, [C.POINTER(GemmNtArgs), _vp]),
    "sgf_gemm_tn_ws_bytes": (C.c_int, [_i32, _i32, _i64, C.POINTER(_sz)]),
    "sgf_gemm_tn": (C.c_int, [C.POINTER(GemmTnArgs), _vp]),
    "sgf_reduce_ws_bytes": (C.c_int, [_i32, C.POINTER(_sz)]),
    "sgf_colstats": (C.c_int, [_vp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sgf_ln_fwd": (C.c_int, [_vp, _vp, _i64, _i64, C.c_int, C.c_int, _f32, _f32, _vp, _vp, C.c_int, C.c_int, _f32,
                             _u64, _vp, _vp, _vp]),
    "sgf_ln_bwd": (C.c_int, [_vp, _vp, _vp, _i64, _i64, C.c_int, C.c_int, _f32, _f32, _vp, _vp, _vp, C.c_int, C.c_int,
                             _f32, _u64, _f32, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sgf_ln_bwd_attn": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, C.c_int, C.c_int, _f32, _f32, _vp, _vp, _vp, C.c_int, C.c_int,
                                  _f32, _u64, _f32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sgf_ln_fwd_graph": (C.c_int, [_vp, _vp, _vp, _i64, _i64, C.c_int, C.c_int, _f32, _f32, _f32, _vp, _vp, C.c_int, C.c_int,
                                   _f32, _u64, _vp, _vp, _vp]),
    "sgf_ln_bwd_attn_graph": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, C.c_int, C.c_int, _f32, _f32, _f32, _vp, _vp, _vp,
                                        C.c_int, _f32, _u64, _f32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                        _sz, _vp]),
    "sgf_gram_ws_bytes": (C.c_int, [_i32, _i32, _i64, C.POINTER(_sz)]),
    "sgf_gram": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _i64, _vp, _i64, _vp, _vp, _sz, _vp]),
    "sgf_attn_gram_ws_floats": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(_i64)]),
    "sgf_attn_gram_prepare_fwd": (C.c_int, [C.POINTER(AttnGramArgs), _vp]),
    "sgf_attn_gram_prepare_bwd": (C.c_int, [C.POINTER(AttnGramArgs), _vp]),
    "sgf_attn_gram_prepare_fwd_vsum": (C.c_int, [C.POINTER(AttnGramArgs), _vp]),
    "sgf_attn_gram_prepare_bwd_vsum": (C.c_int, [C.POINTER(AttnGramArgs), _vp]),
    "sgf_adam_step": (C.c_int, [C.POINTER(AdamArgs), _vp]),
    "sgf_bn_finalize": (C.c_int, [_vp, _vp, _i64, C.c_int, _f32, _f32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sgf_bn_fwd": (C.c_int, [_vp, _vp, _vp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_int, C.c_int,
                             _f32, _u64, _f32, _vp, _vp, _vp, _vp]),
    "sgf_bn_bwd_reduce": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_int,
                                    C.c_int, _f32, _u64, _f32, _vp, _vp, _sz, _vp]),
    "sgf_bn_bwd_apply": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_int,
                                   C.c_int, C.c_int, _f32, _u64, _f32, _i64, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp, _sz, _vp]),
    "sgf_bn_fwd_jk": (C.c_int, [_vp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_int, C.c_int, _f32, _u64, _vp,
                                C.c_int, _vp, _i64, _vp, C.c_int, _vp]),
    "sgf_bn_bwd_reduce_jk": (C.c_int, [_vp, _vp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_int, C.c_int, _f32,
                                       _u64, _vp, C.c_int, _vp, _i64, _vp, C.c_int, _vp, _sz, _vp]),
    "sgf_bn_bwd_apply_jk": (C.c_int, [_vp, _vp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_int, C.c_int,
                                      C.c_int, _f32, _u64, _vp, _vp, _vp, _vp, C.c_int, _vp, _i64, _vp, C.c_int, _vp, _sz, _vp]),
    "sgf_axpby": (C.c_int, [_vp, _i64, C.c_int, _vp, _i64, C.c_int, _f32, _f32, _vp, _vp, _i64, C.c_int, _i64, C.c_int,
                            _vp]),
    "sgf_pack_operand": (C.c_int, [_vp, _i64, _i64, C.c_int, C.c_int, _vp, _i64, C.c_int, _i64, _vp, _vp, _vp, _sz, _vp]),
    "sgf_csr_subset_ws_bytes": (C.c_int, [_i64, _i64, C.POINTER(_sz)]),
    "sgf_csr_subset": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _sz, _vp]),
    "sgf_eval_acc": (C.c_int, [_vp, _i64, _vp, _vp, _i64, _i64, C.c_int, _vp, _vp, _vp]),
    "sgf_softmax_nll": (C.c_int, [_vp, _i64, _vp, _vp, _i64, C.c_int, _f32, _vp, _vp, _i64, _vp, _sz, _vp]),
    "sgf_head_mean": (C.c_int, [_vp, _i64, _i64, C.c_int, C.c_int, C.c_int, _vp, _i64, _vp]),
    "sgf_attn_prepare_fwd": (C.c_int, [_vp, _vp, _vp, C.c_int, _vp, C.c_int, C.c_int, C.c_int, _vp, _i64, _vp, _i64,
                                       _i64, _vp, _vp]),
    "sgf_attn_bwd_prep": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i64, C.c_int, C.c_int, _f32, _vp, _i64, _vp, _vp]),
    "sgf_attn_combine_scal": (C.c_int, [_vp, C.c_int, C.c_int, _vp, _vp]),
    "sgf_gat_logits": (C.c_int, [_vp, _i64, _i64, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp]),
    "sgf_gat_fwd": (C.c_int, [_vp, _vp, _vp, _i64, _vp, _vp, _i64, C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp, _i64, _vp, _f32,
                              _u64, _vp]),
    "sgf_gat_bwd": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i64, C.c_int, C.c_int, C.c_int,
                              C.c_int, _f32, _u64, _vp, _vp, _vp, _vp, _i64, _vp]),
    "sgf_dense_dropout": (C.c_int, [_vp, _i64, _i64, _i64, _f32, _u64, _vp, _i64, _vp]),
    "sgf_csr_build_weighted_ws_bytes": (C.c_int, [_i64, _i64, C.POINTER(_sz)]),
    "sgf_csr_build_weighted": (C.c_int, [_vp, _vp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sgf_edge_symmetry_weighted": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _vp]),
    "sgf_spmm_weighted": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _i64, C.c_int, C.c_int, _i64, _vp]),
    "sgf_spmm_heavy_weighted": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _i64, C.c_int, C.c_int, _vp, _vp, _i64, _vp, _vp, _vp,
                                          _i64, _vp]),
    "sgf_spmm_sum": (C.c_int, [_vp, _vp, _vp, _i64, _vp, _i64, _i64, C.c_int, C.c_int, _i64, _vp]),
    "sgf_spmm_heavy_sum": (C.c_int, [_vp, _vp, _i64, _vp, _i64, C.c_int, C.c_int, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _vp]),
    "sgf_edge_weight_grad": (C.c_int, [_vp, _vp, _vp, _i64, C.c_int, C.c_int, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp,
                                       _vp, _i64, _vp, _vp, _vp]),
    "sgf_attn_prepare_bwd": (C.c_int, [_vp, _vp, _vp, _vp, _vp, C.c_int, C.c_int, _vp, _i64, _vp, _i64, _vp, _i64, _i64,
                                       _i64, _vp, _vp, _vp, _vp]),
}

_lib = None


def lib_path():
    return _build.LIB_PATH


def load():
    """Load (once) and return the ctypes handle; raises if the library has not been built."""
    global _lib
    if _lib is None:
        path = lib_path()
        if not os.path.exists(path):
            raise RuntimeError(
                f"sgformer_b200: CUDA library not built ({path} missing). Run `python -c 'import __graft_entry__ as g; "
                "g.build()'` at the repo root. There is no CPU fallback.")
        lib = C.CDLL(path)
        for name, (res, args) in _SIGS.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is missing: fail loudly
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


_CUDA_ERRORS = {1: "invalid value", 2: "out of memory", 98: "invalid device function", 209: "no kernel image for device",
                700: "illegal address", 701: "launch out of resources", 716: "misaligned address", 719: "launch failure",
                35: "driver too old", 100: "no CUDA device", 101: "invalid device"}


def check(rc, what):
    if rc == 0:
        return
    if rc < 0:
        kind = {-1: "invalid argument", -2: "unsupported shape", -3: "driver entry point / tensor-map failure"}.get(rc, "?")
        raise RuntimeError(f"sgformer_b200: {what} failed: {kind} (code {rc})")
    raise RuntimeError(f"sgformer_b200: {what} failed: CUDA error {rc} ({_CUDA_ERRORS.get(rc, 'see cudaError_t')})")
