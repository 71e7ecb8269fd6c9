"""ctypes loader for libnova_b200.so.  Fails loudly -- there is no fallback path."""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

c_size_t, c_int, c_void_p, c_u64 = ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64


# status codes of include/nova_b200.h
B200_OK, B200_E_ARG, B200_E_CUDA, B200_E_HANDLE, B200_E_NOMEM, B200_E_RANGE = 0, 1, 2, 3, 4, 5
B200_E_ZERO, B200_E_POINT, B200_E_PEER, B200_E_INDEX = 6, 7, 8, 9
ERROR_NAMES = {B200_E_ARG: "B200_E_ARG", B200_E_CUDA: "B200_E_CUDA", B200_E_HANDLE: "B200_E_HANDLE",
               B200_E_NOMEM: "B200_E_NOMEM", B200_E_RANGE: "B200_E_RANGE", B200_E_ZERO: "B200_E_ZERO",
               B200_E_POINT: "B200_E_POINT", B200_E_PEER: "B200_E_PEER", B200_E_INDEX: "B200_E_INDEX"}


class B200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"nova_b200 error {code}: {msg}")
        self.code = code
        self.name = ERROR_NAMES.get(code, "unknown")


def library_path() -> str:
    # NOVA_B200_LIB selects another build of the same library (A/B timing of kernel variants)
    return os.environ.get("NOVA_B200_LIB") or os.path.join(_HERE, "libnova_b200.so")


# every symbol include/nova_b200.h declares: name -> argtypes (all return int unless noted)
_P = c_void_p
SIGNATURES = {
    "b200_init": [c_int],
    "b200_device_count": [ctypes.POINTER(c_int)],
    "b200_host_alloc": [c_size_t, ctypes.POINTER(_P)],
    "b200_host_free": [_P],
    "b200_dev_alloc": [c_size_t, ctypes.POINTER(_P)],
    "b200_dev_free": [_P],
    "b200_memcpy_h2d": [_P, _P, c_size_t],
    "b200_memcpy_d2h": [_P, _P, c_size_t],
    "b200_memcpy_d2d": [_P, _P, c_size_t, _P],
    "b200_memset_dev": [_P, c_int, c_size_t, _P],
    "b200_sync": [],
    "b200_profile_enable": [c_int],
    "b200_profile_reset": [],
    "b200_profile_read": [ctypes.POINTER(ctypes.c_double), c_int, ctypes.POINTER(c_u64), ctypes.POINTER(c_u64)],
    "b200_jacobian_sum_dev": [c_int, _P, c_size_t, _P, _P],
    "b200_ck_register": [c_int, _P, c_size_t, _P, c_int, ctypes.POINTER(c_u64)],
    "b200_ck_register_checked": [c_int, _P, c_size_t, _P, c_int, ctypes.POINTER(c_u64), ctypes.POINTER(c_size_t)],
    "b200_ck_setup_synthetic": [c_int, _P, c_u64, c_size_t, c_int, c_int, ctypes.POINTER(c_u64)],
    "b200_poseidon_register": [c_int, c_int, c_int, c_int, _P, _P, ctypes.POINTER(c_u64)],
    "b200_poseidon_release": [c_u64],
    "b200_poseidon_ro": [c_u64, _P, c_size_t, c_int, c_int, _P],
    "b200_poseidon_ro_dev": [c_u64, _P, c_size_t, c_int, c_int, _P, _P],
    "b200_to_mont_dev": [c_int, _P, c_size_t, _P, _P],
    "b200_mgpu_init": [c_int, ctypes.POINTER(c_int)],
    "b200_mgpu_ck_register": [c_int, _P, c_size_t, _P, c_int, ctypes.POINTER(c_u64)],
    "b200_mgpu_ck_release": [c_u64],
    "b200_mgpu_commit": [c_u64, _P, c_size_t, _P, _P],
    "b200_keccak256": [_P, c_size_t, _P],
    "b200_peer_buffer_alloc": [ctypes.POINTER(_P)],
    "b200_peer_buffer_free": [_P],
    "b200_ipc_export": [_P, _P],
    "b200_ipc_open": [_P, ctypes.POINTER(_P)],
    "b200_ipc_close": [_P],
    "b200_peer_group_create": [c_int, c_int, ctypes.POINTER(_P), ctypes.POINTER(c_u64)],
    "b200_peer_group_release": [c_u64],
    "b200_peer_group_status": [c_u64],
    "b200_msm_sharded_dev": [c_u64, c_size_t, _P, c_size_t, c_u64, _P, _P],
    "b200_ck_setup_tau": [c_int, _P, _P, c_size_t, c_int, ctypes.POINTER(c_u64)],
    "b200_ck_export_bases": [c_u64, c_size_t, c_size_t, _P],
    "b200_ck_derive_by_address": [c_u64, ctypes.POINTER(c_u64), c_size_t, c_size_t, c_int, ctypes.POINTER(c_u64),
                                  ctypes.POINTER(c_size_t)],
    "b200_ck_derive_by_address_dev": [c_u64, _P, c_size_t, c_size_t, c_int, ctypes.POINTER(c_u64),
                                      ctypes.POINTER(c_size_t), _P],
    "b200_ck_release": [c_u64],
    "b200_ck_len": [c_u64, ctypes.POINTER(c_size_t), ctypes.POINTER(c_int), ctypes.POINTER(c_int)],
    "b200_msm": [c_u64, c_size_t, _P, c_size_t, _P],
    "b200_msm_dev": [c_u64, c_size_t, _P, c_size_t, _P, _P],
    "b200_commit": [c_u64, _P, c_size_t, _P, _P],
    "b200_commit_dev": [c_u64, _P, c_size_t, _P, _P, _P],
    "b200_commit_many_dev": [c_u64, ctypes.POINTER(_P), ctypes.POINTER(c_size_t), c_size_t, _P, _P],
    "b200_msm_many_dev": [c_u64, ctypes.POINTER(c_size_t), ctypes.POINTER(_P), ctypes.POINTER(c_size_t), c_size_t, _P, _P],
    "b200_fold_halves_dev": [c_int, _P, c_size_t, _P, _P, _P, _P],
    "b200_ipa_scalars_dev": [c_int, _P, _P, c_size_t, c_size_t, _P, _P, _P],
    "b200_ipa_weights_dev": [c_int, _P, c_size_t, c_size_t, _P, _P, _P],
    "b200_ipa_s_dev": [c_int, _P, _P, c_int, _P, _P, _P],
    "b200_msm_batch": [c_u64, ctypes.POINTER(_P), ctypes.POINTER(c_size_t), c_size_t, _P],
    "b200_msm_small": [c_u64, c_size_t, _P, c_int, c_size_t, c_int, _P],
    "b200_msm_indices": [c_u64, ctypes.POINTER(c_u64), c_size_t, _P],
    "b200_msm_adhoc": [c_int, _P, _P, c_size_t, _P],
    "b200_cross_term": [c_int, _P, _P, _P, _P, _P, _P, c_size_t, _P],
    "b200_axpy": [c_int, _P, _P, _P, c_size_t, _P],
    "b200_vec_add": [c_int, _P, _P, c_size_t, _P],
    "b200_bind_top": [c_int, _P, c_size_t, _P],
    "b200_cross_term_dev": [c_int, _P, _P, _P, _P, _P, _P, c_size_t, _P, _P],
    "b200_axpy_dev": [c_int, _P, _P, _P, c_size_t, _P, _P],
    "b200_vec_add_dev": [c_int, _P, _P, c_size_t, _P, _P],
    "b200_vec_mul_dev": [c_int, _P, _P, c_size_t, _P, _P],
    "b200_logup_hash_dev": [c_int, _P, _P, _P, _P, c_size_t, _P, _P],
    "b200_bind_top_dev": [c_int, _P, c_size_t, _P, _P],
    "b200_bind_top_multi_dev": [c_int, ctypes.POINTER(_P), c_size_t, c_size_t, _P, _P],
    "b200_sc_eval": [c_int, c_int, _P, _P, _P, c_size_t, _P, c_size_t, _P, c_size_t, c_int, _P],
    "b200_sc_eval_dev": [c_int, c_int, _P, _P, _P, c_size_t, _P, _P, c_int, _P, _P],
    "b200_sc_eval_sharded_dev": [c_int, c_int, _P, _P, _P, c_size_t, _P, _P, c_int, c_size_t, c_size_t, _P, _P],
    "b200_ck_validate": [c_int, _P, c_size_t, ctypes.POINTER(c_size_t)],
    "b200_witness_begin": [c_u64, c_size_t, ctypes.POINTER(c_u64)],
    "b200_witness_append": [c_u64, _P, c_size_t],
    "b200_witness_finish": [c_u64, _P, _P, ctypes.POINTER(_P)],
    "b200_witness_reset": [c_u64],
    "b200_witness_release": [c_u64],
    "b200_sc_round_dev": [c_int, c_int, _P, _P, _P, _P, _P, c_size_t, c_int, c_int, _P, _P, _P],
    "b200_sc_round_batched_dev": [c_int, _P, _P, _P, _P, c_size_t, c_int, c_int, _P, _P, _P],
    "b200_sumcheck_quad_prod": [c_int, _P, c_int, _P, _P, _P, _P, c_size_t, _P, _P, _P],
    "b200_sumcheck_cubic3": [c_int, _P, _P, c_int, _P, _P, _P, _P, _P, c_size_t, _P, _P, _P],
    "b200_sumcheck_tail_bits": [c_int],
    "b200_sumcheck_batched": [c_int, _P, _P, _P, _P, _P, _P, c_size_t, _P, _P, _P],
    "b200_eq_table": [c_int, _P, c_int, _P],
    "b200_eq_table_dev": [c_int, _P, c_int, _P, _P],
    "b200_mle_eval": [c_int, _P, c_int, _P, _P],
    "b200_mle_eval_dev": [c_int, _P, c_int, _P, _P, _P],
    "b200_mle_eval_multi_dev": [c_int, _P, c_size_t, c_int, _P, _P, _P],
    "b200_batch_invert": [c_int, _P, c_size_t, _P],
    "b200_batch_invert_dev": [c_int, _P, c_size_t, _P, _P, _P],
    "b200_rlc": [c_int, ctypes.POINTER(_P), ctypes.POINTER(c_size_t), c_size_t, _P, c_size_t, _P],
    "b200_rlc_dev": [c_int, ctypes.POINTER(_P), ctypes.POINTER(c_size_t), c_size_t, _P, c_size_t, _P, _P],
    "b200_kzg_fold": [c_int, _P, c_size_t, _P, _P],
    "b200_kzg_fold_dev": [c_int, _P, c_size_t, _P, _P, _P],
    "b200_poly_eval": [c_int, _P, c_size_t, _P, c_size_t, _P],
    "b200_poly_eval_dev": [c_int, _P, c_size_t, _P, c_size_t, _P, _P],
    "b200_poly_eval_many_dev": [c_int, _P, _P, c_size_t, _P, c_size_t, _P, _P],
    "b200_poly_div": [c_int, _P, c_size_t, _P, _P],
    "b200_poly_div_dev": [c_int, _P, c_size_t, _P, _P, _P],
    "b200_mat_vec_rows": [c_int, _P, c_size_t, c_size_t, _P, _P],
    "b200_mat_vec_rows_dev": [c_int, _P, c_size_t, c_size_t, _P, _P, _P],
    "b200_div_binomial": [c_int, _P, c_size_t, c_size_t, _P, _P, _P],
    "b200_div_binomial_dev": [c_int, _P, c_size_t, c_size_t, _P, _P, _P, _P],
    "b200_mercury_s_poly": [c_int, _P, _P, _P, _P, c_size_t, _P, _P],
    "b200_mercury_s_poly_dev": [c_int, _P, _P, _P, _P, c_size_t, _P, _P, _P],
    "b200_neutron_evals": [c_int] + [_P] * 8 + [c_size_t, c_size_t, _P],
    "b200_neutron_evals_dev": [c_int] + [_P] * 8 + [c_size_t, c_size_t, _P, _P],
    "b200_pow_split_evals": [c_int, _P, c_size_t, c_size_t, _P],
    "b200_pow_split_evals_dev": [c_int, _P, c_size_t, c_size_t, _P, _P],
    "b200_lerp": [c_int, _P, _P, _P, c_size_t, _P],
    "b200_lerp_dev": [c_int, _P, _P, _P, c_size_t, _P, _P],
    "b200_spmv_register": [c_int, _P, ctypes.POINTER(c_u64), ctypes.POINTER(c_u64), c_size_t, c_size_t,
                           ctypes.POINTER(c_u64)],
    "b200_spmv_release": [c_u64],
    "b200_spmv_dev": [c_u64, _P, _P, _P, _P, _P],
    "b200_spmv_t": [c_u64, _P, c_size_t, _P],
    "b200_spmv_t_dev": [c_u64, _P, c_size_t, _P, _P],
    "b200_gather": [_P, c_size_t, ctypes.POINTER(c_u64), c_size_t, _P],
    "b200_gather_dev": [_P, _P, c_size_t, _P, _P],
    "b200_spark_repr_dev": [c_u64, c_u64, c_u64, c_size_t, ctypes.POINTER(_P), _P, _P, _P],
    "b200_r1cs_eval_dev": [ctypes.POINTER(c_u64), c_size_t, _P, c_size_t, _P, c_size_t, _P, _P],
    "b200_r1cs_eval": [ctypes.POINTER(c_u64), c_size_t, _P, c_int, _P, c_int, _P],
    "b200_spmv_multi": [ctypes.POINTER(c_u64), c_size_t, _P, _P, c_size_t, ctypes.POINTER(_P),
                        ctypes.POINTER(_P)],
}
STRING_FUNCS = ["b200_last_error", "b200_version"]


def lib():
    """Load the C-ABI library (does not touch the GPU)."""
    global _LIB
    if _LIB is None:
        path = library_path()
        if not os.path.exists(path):
            raise ImportError(
                f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "or `make -C nova_b200/csrc`.  nova_b200 has no CPU fallback."
            )
        L = ctypes.CDLL(path)
        for name, args in SIGNATURES.items():
            fn = getattr(L, name)
            fn.argtypes = args
            fn.restype = c_int
        for name in STRING_FUNCS:
            getattr(L, name).restype = ctypes.c_char_p
            getattr(L, name).argtypes = []
        _LIB = L
    return _LIB


def check(rc: int):
    if rc != 0:
        raise B200Error(rc, lib().b200_last_error().decode())
