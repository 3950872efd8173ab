"""ctypes binding of libnlam_b200.so (C ABI in include/nlam_b200.h).

The library is the product: there is no CPU or eager-PyTorch fallback.  Import succeeds
without a GPU (so that the host logic can be tested), but every compute entry point raises
if the CUDA extension is missing or fails.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libnlam_b200.so")

NLAM_MAX_LINEAR = 4
NLAM_MAX_SRC = 4

AGGR_MEAN = 0x1
PROPAGATION = 0x2
MATH_TF32 = 0x10
MATH_FP32 = 0x20
HINT_ONE_HIDDEN = 0x100
EDGE_ONLY = 0x200
E_UNSUPPORTED = 2  # NLAM_E_UNSUPPORTED

c_float_p = ctypes.c_void_p  # device pointers travel as integers
c_int32_p = ctypes.c_void_p


class NlamMlp(ctypes.Structure):
    _fields_ = [
        ("n_linear", ctypes.c_int32),
        ("in_dim", ctypes.c_int32),
        ("out_dim", ctypes.c_int32 * NLAM_MAX_LINEAR),
        ("w", ctypes.c_void_p * NLAM_MAX_LINEAR),
        ("b", ctypes.c_void_p * NLAM_MAX_LINEAR),
        ("ln_gamma", ctypes.c_void_p),
        ("ln_beta", ctypes.c_void_p),
        ("ln_eps", ctypes.c_float),
        ("_pad", ctypes.c_int32),
    ]


class NlamRowSrc(ctypes.Structure):
    _fields_ = [
        ("ptr", ctypes.c_void_p),
        ("idx", ctypes.c_void_p),
        ("bstride", ctypes.c_int64),
        ("dim", ctypes.c_int32),
        ("_pad", ctypes.c_int32),
    ]


class NlamMlpGrads(ctypes.Structure):
    _fields_ = [
        ("w", ctypes.c_void_p * NLAM_MAX_LINEAR),
        ("b", ctypes.c_void_p * NLAM_MAX_LINEAR),
        ("ln_gamma", ctypes.c_void_p),
        ("ln_beta", ctypes.c_void_p),
    ]


class NlamError(RuntimeError):
    pass


_lib = None

# name -> (restype, argtypes); every symbol include/nlam_b200.h declares
SYMBOLS = {
    "nlam_abi_version": (ctypes.c_int, []),
    "nlam_last_error": (ctypes.c_char_p, []),
    "nlam_build_info": (ctypes.c_char_p, []),
    "nlam_launch_count": (ctypes.c_int64, []),
    "nlam_profile_enable": (None, [ctypes.c_int]),
    "nlam_profile_count": (ctypes.c_int, []),
    "nlam_profile_get": (ctypes.c_int, [ctypes.c_int, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(ctypes.c_float),
                                        ctypes.POINTER(ctypes.c_double)]),
    "nlam_graph_create": (ctypes.c_int, [ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int]),
    "nlam_graph_destroy": (None, [ctypes.c_void_p]),
    "nlam_graph_num_edges": (ctypes.c_int64, [ctypes.c_void_p]),
    "nlam_graph_num_rec": (ctypes.c_int64, [ctypes.c_void_p]),
    "nlam_graph_num_send": (ctypes.c_int64, [ctypes.c_void_p]),
    "nlam_graph_max_in_degree": (ctypes.c_int32, [ctypes.c_void_p]),
    "nlam_graph_is_sorted": (ctypes.c_int32, [ctypes.c_void_p]),
    "nlam_graph_uniform_degree": (ctypes.c_int32, [ctypes.c_void_p]),
    "nlam_graph_rowptr": (ctypes.c_void_p, [ctypes.c_void_p]),
    "nlam_graph_src": (ctypes.c_void_p, [ctypes.c_void_p]),
    "nlam_graph_dst": (ctypes.c_void_p, [ctypes.c_void_p]),
    "nlam_graph_perm": (ctypes.c_void_p, [ctypes.c_void_p]),
    "nlam_graph_inv_perm": (ctypes.c_void_p, [ctypes.c_void_p]),
    "nlam_graph_sptr": (ctypes.c_void_p, [ctypes.c_void_p]),
    "nlam_graph_sperm": (ctypes.c_void_p, [ctypes.c_void_p]),
    "nlam_inet_workspace_bytes": (ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "nlam_inet_chain_supported": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp), ctypes.c_void_p,
                                                 ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
                                                 ctypes.c_int]),
    "nlam_inet_fwd_chain": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp), ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
        ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "nlam_inet_inplace_supported": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(NlamMlp), ctypes.c_void_p, ctypes.c_int64,
                                                   ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
                                                   ctypes.c_int, ctypes.c_int]),
    "nlam_inet_fwd": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp),
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
        ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "nlam_rowmlp_fwd": (ctypes.c_int, [
        ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamRowSrc), ctypes.c_int, ctypes.POINTER(NlamRowSrc),
        ctypes.POINTER(NlamRowSrc), ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
        ctypes.c_int, ctypes.c_void_p]),
    "nlam_segment_sum": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "nlam_gather_rows": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "nlam_rowmlp_step_fwd": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
        ctypes.c_void_p]),
    "nlam_rowmlp_step_std_fwd": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
        ctypes.c_void_p]),
    "nlam_step_epilogue_clamped": (ctypes.c_int, [ctypes.c_void_p] * 10 + [ctypes.c_int64] * 3 + [ctypes.c_void_p]),
    "nlam_halo_push": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "nlam_linear": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                    ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "nlam_pack_rows": (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int] * 4 + [ctypes.c_int64] * 4 +
                       [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p]),
    "nlam_mlp_bwd_workspace_bytes": (ctypes.c_size_t, [ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamRowSrc), ctypes.c_int,
                                                       ctypes.c_int64, ctypes.c_int]),
    "nlam_mlp_bwd": (ctypes.c_int, [ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamRowSrc), ctypes.c_int, ctypes.c_void_p,
                                    ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(NlamMlpGrads), ctypes.c_int64, ctypes.c_int,
                                    ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "nlam_inet_bwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "nlam_inet_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp), ctypes.c_void_p,
                                     ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
                                     ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                     ctypes.POINTER(NlamMlpGrads), ctypes.POINTER(NlamMlpGrads), ctypes.c_int, ctypes.c_int,
                                     ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "nlam_silu": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]),
    "nlam_layernorm_fwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p]),
    "nlam_layernorm_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "nlam_bwd_scratch_floats": (ctypes.c_size_t, [ctypes.c_int]),
    "nlam_colsum": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "nlam_reduce_partials": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p]),
    "nlam_transpose_pad": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]),
    "nlam_add_gather": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "nlam_memcpy2d_async": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t,
                                            ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]),
    "nlam_node_update_step_fwd": (ctypes.c_int, [
        ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp), ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
        ctypes.c_int, ctypes.c_void_p]),
    "nlam_node_update_step_std_fwd": (ctypes.c_int, [
        ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp), ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "nlam_decode_workspace_bytes": (ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int]),
    "nlam_decode_step_fwd": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp),
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "nlam_decode_step_std_fwd": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp),
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "nlam_encode_supported": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamRowSrc), ctypes.c_int, ctypes.POINTER(NlamMlp),
        ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp), ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int]),
    "nlam_encode_fwd": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamRowSrc), ctypes.c_int, ctypes.POINTER(NlamMlp),
        ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp), ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
        ctypes.c_void_p]),
    "nlam_latent_sample_supported": (ctypes.c_int, [
        ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp), ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int]),
    "nlam_latent_sample_fwd": (ctypes.c_int, [
        ctypes.POINTER(NlamMlp), ctypes.POINTER(NlamMlp), ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64,
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "nlam_memcpy3d_async": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                            ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int,
                                            ctypes.c_void_p]),
    "nlam_ensemble_stats_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int64, ctypes.c_int]),
    "nlam_ensemble_stats": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_int,
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "nlam_ensemble_stats_bwd": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_int,
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "nlam_step_epilogue": (ctypes.c_int, [
        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p]),
}


def lib():
    """Load the shared library (once).  Raises NlamError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise NlamError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / eager fallback)"
        )
    L = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(L, name)  # AttributeError if the .so is stale
        fn.restype = res
        fn.argtypes = args
    if L.nlam_abi_version() != 3:
        raise NlamError("libnlam_b200.so ABI version mismatch; rebuild")
    _lib = L
    return L


def check(rc):
    if rc != 0:
        msg = lib().nlam_last_error()
        raise NlamError(f"libnlam_b200 error {rc}: {msg.decode() if msg else '?'}")
