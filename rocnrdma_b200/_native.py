"""ctypes binding to ``lib/librocnrdma_b200.so`` (the flat ``rn_*`` C ABI).

The library is built in-tree by :mod:`rocnrdma_b200.build`.  If it is missing and
nvcc is available it is built on first use; on a GPU box a missing library is a
hard error -- there is no Python fallback for the data path.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_LIB = None
_LIB_PATH = Path(__file__).resolve().parent / "lib" / "librocnrdma_b200.so"

u8, u16, u32, u64, i32 = C.c_uint8, C.c_uint16, C.c_uint32, C.c_uint64, C.c_int
vp = C.c_void_p


class NativeError(RuntimeError):
    pass


class RnWc(C.Structure):
    _fields_ = [("qpn", u32), ("byte_cnt", u32), ("imm", u32), ("wqe_counter", u16),
                ("opcode", u8), ("syndrome", u8), ("wqe_opcode", u8), ("is_error", u8)]


class RnRemote(C.Structure):
    _fields_ = [("rkeys", u64), ("n_rkeys", u32), ("qpn", u32), ("rq", u64), ("rq_dbr", u64),
                ("rq_log", u32), ("pad", u32), ("rcq", u64), ("rcq_buf", u64)]


class RnQpCounters(C.Structure):
    _fields_ = [("n_wqe", u64), ("n_cqe", u64), ("n_err", u64), ("n_db_order_violations", u64),
                ("n_bytes", u64), ("n_rnr", u64), ("resv_head", u64), ("ready_head", u64),
                ("sq_cons", u64), ("cursor", u64), ("retire_head", u64), ("state", u32), ("pad", u32),
                ("n_fence_waits", u64)]


class RnVWc(C.Structure):
    _fields_ = [("wr_id", u64), ("status", u32), ("opcode", u32), ("byte_len", u32), ("imm", u32), ("qp_num", u32),
                ("vendor_err", u32), ("with_imm", u32), ("pad", u32)]


class RnRawQp(C.Structure):
    _fields_ = [("sq_buf", u64), ("sq_wqe_cnt", u32), ("sq_stride", u32), ("rq_buf", u64), ("rq_wqe_cnt", u32), ("rq_stride", u32),
                ("dbrec", u64), ("bf_reg", u64), ("bf_size", u32), ("qpn", u32),
                ("cq_buf", u64), ("cq_cqe_cnt", u32), ("cq_cqe_size", u32), ("cq_dbrec", u64), ("cqn", u32), ("pad0", u32),
                ("rcq_buf", u64), ("rcq_cqe_cnt", u32), ("rcq_cqe_size", u32), ("rcq_dbrec", u64), ("rcqn", u32), ("pad1", u32)]


class RnGpuQp(C.Structure):
    _fields_ = [("sq_dev", u64), ("rq_dev", u64), ("dbrec_dev", u64), ("bf_dev", u64), ("cq_dev", u64), ("cq_dbrec_dev", u64),
                ("rcq_dev", u64), ("rcq_dbrec_dev", u64), ("sq_wqe_cnt", u32), ("rq_wqe_cnt", u32), ("cq_cqe_cnt", u32),
                ("rcq_cqe_cnt", u32), ("qpn", u32), ("cqn", u32), ("rcqn", u32), ("flags", u32)]


class RnMockQpStats(C.Structure):
    _fields_ = [("n_wqe", u64), ("n_cqe", u64), ("n_err", u64), ("n_bytes", u64), ("n_rnr", u64), ("n_db_no_progress", u64),
                ("n_doorbells", u64), ("hw_sq_cons", u64), ("sq_cq_overruns", u64)]


class RnSge(C.Structure):
    """One scatter-gather entry (``rn::Sge``): ``bytes`` at ``addr`` under ``lkey``."""
    _fields_ = [("addr", u64), ("lkey", u32), ("bytes", u32)]


class RnEngineStats(C.Structure):
    _fields_ = [("n_bulk_chunks", u64), ("t_start", u64), ("t_exit", u64), ("running_ctas", u32),
                ("exited_idle", u32), ("fatal", u32), ("n_qps", u32), ("ctas", u32), ("pad", u32)]


_SIGS = {
    "rn_last_error": (C.c_char_p, []),
    "rn_abi_sizes": (i32, [C.POINTER(u32), i32]),
    "rn_hca_open": (i32, [i32, u32, u32, u64, u64, C.POINTER(vp)]),
    "rn_hca_close": (i32, [vp]),
    "rn_hca_mkey_table": (u64, [vp]),
    "rn_hca_arena": (u64, [vp, C.POINTER(u64)]),
    "rn_classify_ptr": (i32, [u64, C.POINTER(i32)]),
    "rn_reg_mr": (i32, [vp, u64, u64, u32, C.POINTER(u32)]),
    "rn_reg_mr_mode": (i32, [vp, u64, u64, u32, u32, C.POINTER(u32), C.POINTER(i32)]),
    "rn_mr_revoke": (i32, [vp, u32]),
    "rn_dereg_mr": (i32, [vp, u32]),
    "rn_mr_state": (i32, [vp, u32]),
    "rn_create_cq": (i32, [vp, u32, u32, C.POINTER(vp)]),
    "rn_cq_dev": (u64, [vp]),
    "rn_poll_cq": (i32, [vp, i32, C.POINTER(RnWc)]),
    "rn_create_qp": (i32, [vp, vp, vp, u32, u32, u32, u32, C.POINTER(vp)]),
    "rn_qp_dev": (u64, [vp]),
    "rn_qp_num": (u32, [vp]),
    "rn_qp_set_flags": (i32, [vp, i32, i32]),
    "rn_qp_read_trace": (i32, [vp, C.POINTER(u64), u32]),
    "rn_qp_state": (u32, [vp]),
    "rn_qp_describe": (i32, [vp, C.POINTER(RnRemote)]),
    "rn_qp_connect": (i32, [vp, C.POINTER(RnRemote)]),
    "rn_modify_qp": (i32, [vp, u32]),
    "rn_qp_connect_pair": (i32, [vp, vp]),
    "rn_qp_query": (i32, [vp, C.POINTER(RnQpCounters)]),
    "rn_post_send": (i32, [vp, u32, u64, u32, u64, u32, u32, u32, u32, C.POINTER(u64)]),
    "rn_post_recv": (i32, [vp, u64, u32, u32]),
    "rn_post_atomic": (i32, [vp, u32, u64, u32, u64, u32, u64, u64, u32, C.POINTER(u64)]),
    "rn_post_inline": (i32, [vp, u32, u64, u32, vp, u32, u32, u32, C.POINTER(u64)]),
    "rn_post_wqe_bytes": (i32, [vp, C.POINTER(u8), C.POINTER(u64)]),
    "rn_post_send_sg": (i32, [vp, u32, C.POINTER(RnSge), i32, u64, u32, u32, u32, C.POINTER(u64)]),
    "rn_hca_host_native_atomics": (i32, [vp]),
    "rn_host_stream": (i32, [vp, u32, u64, u32, u64, u32, u32, u32, u32, u64, u32, u64, C.POINTER(u64), C.POINTER(u32)]),
    "rn_host_staged_stream": (i32, [vp, u64, u64, u64, u32, u64, u32, u32, u32, u64, u32, u64, C.POINTER(u64)]),
    "rn_engine_running": (i32, [vp]),
    "rn_engine_start": (i32, [vp, i32, u64, u64]),
    "rn_engine_stop": (i32, [vp]),
    "rn_engine_set_oneshot": (i32, [vp, i32]),
    "rn_engine_wait": (i32, [vp]),
    "rn_engine_stats": (i32, [vp, C.POINTER(RnEngineStats)]),
    "rn_engine_mover_profile": (i32, [vp, C.POINTER(u64), i32]),
    "rn_k_engine_ceiling": (i32, [u64, u64, u64, u64, i32, u64, u64]),
    "rn_hca_scratch": (u64, [vp, C.POINTER(u64)]),
    "rn_set_device": (i32, [i32]),
    "rn_ipc_export": (i32, [u64, C.POINTER(u8), C.POINTER(u64), C.POINTER(u64)]),
    "rn_ipc_open": (i32, [vp, C.POINTER(u8), C.POINTER(u64)]),
    "rn_ipc_close": (i32, [u64]),
    "rn_hca_alloc_remote_table": (u64, [vp, u32]),
    "rn_hca_set_remote_mkey": (i32, [vp, u64, u32, u64, u64, u64, u32, u32]),
    "rn_hca_work_stream": (u64, [vp]),
    "rn_hca_aux_stream": (u64, [vp]),
    "rn_hca_stream": (u64, [vp, i32]),
    "rn_hca_dev_scratch": (u64, [vp, C.POINTER(u64)]),
    "rn_pack_record_bytes": (u64, [u64]),
    "rn_pack_tile_elems": (u32, []),
    "rn_k_pack_fp8_write": (i32, [u64, i32, u64, u64, u64, u32, u64, u64, u32, u64, u32, u32, u32, u64, u64, u64, u64]),
    "rn_k_pack_fp8_scatter": (i32, [u64, i32, u64, u64, u64, u32, u32, u32, C.POINTER(u64), C.POINTER(u64), C.POINTER(u32),
                                    u64, u32, u64, u64, u32, u32, u64, u64, u64]),
    "rn_gemm_timeline": (i32, [C.POINTER(C.c_uint64)]),
    "rn_k_gemm_send": (i32, [u64, i32, u64, u64, u64, u32, u32, u32, u64, u64, u32, u64, u32, u32, u32, u32, u32, u32, u32, u64, u64, u64]),
    "rn_k_gemm_reduce_send": (i32, [u64, i32, u64, u64, u32, u32, u32, u64, u64, u64, u32, u64, u32, u64, u32, u64, u64, u32, u64,
                                    u64, u32, u64, u32, u32, u32, u32, u32, u64, u64, u64]),
    "rn_k_gemm_mxfp8": (i32, [u64, i32, u64, u64, u32, u64, u64, u64, u32, u64, u64, u32, u32, u32, u64, u32, u64, u64, u64]),
    "rn_k_gemm_mxfp8_ordered": (i32, [u64, i32, u64, u64, u32, u64, u64, u64, u32, u64, u64, u32, u32, u32, u64, u32, u64, u64, u64,
                                      u64]),
    "rn_k_shared_post_stress": (i32, [u64, u64, i32, u64, u32, u64, u32, u32, u64, u64, u64]),
    "rn_k_recv_consume": (i32, [u64, u64, u32, u32, u64, u64, u64, u64, u32, u32]),
    "rn_k_recv_consume_qps": (i32, [u64, C.POINTER(u64), C.POINTER(u32), u32, u32, u32, u64, u64, u64, u64, u32]),
    "rn_hca_enable_peer": (i32, [vp, i32]),
    "rn_k_unpack_fp8": (i32, [u64, i32, u64, u64, u64, u32, u64, u64, u64, u64, u64, u64, u64, u32, u64, u32, u32, u32, u32]),
    "rn_k_relay_records": (i32, [u64, u64, u64, u32, u32, u64, u64, u32, u64, u32, u64, u32, u32, u64, u64, u64]),
    "rn_k_reduce_fp8": (i32, [u64, i32, u64, u32, u64, u64, u64, u64, u32, u64, u64, u64, u32, u64, u32, u32, u32, u64, u64, u64,
                              u32, u64]),
    "rn_k_rdma_stream": (i32, [u64, C.POINTER(u64), u32, u32, u64, u32, u64, u32, u64, u32, u32, u32, u32, u32, u64, u32, u64, u64, u32]),
    "rn_k_write_read": (i32, [u64, u64, u64, u32, u64, u32, u64, u32, u32, u32, u32, u64, u64]),
    "rn_stream_clamp": (None, [u32, C.POINTER(u32), C.POINTER(u32)]),
    "rn_wire_build_wqe": (None, [C.POINTER(u8), u32, u32, u32, u64, u32, u64, u32, u32, u32, u32]),
    "rn_wire_build_cqe": (None, [C.POINTER(u8), u32, u32, u32, u32, u32, u32, u32, u32, u32, u64]),
    "rn_wire_decode_cqe": (i32, [C.POINTER(u8), C.POINTER(RnWc)]),
    "rn_wire_build_atomic_wqe": (None, [C.POINTER(u8), u32, u32, u32, u64, u32, u64, u32, u64, u64, u32]),
    "rn_wire_decode_wqe": (i32, [C.POINTER(u8), C.POINTER(u64)]),
    "rn_wire_build_inline_wqe": (None, [C.POINTER(u8), u32, u32, u32, u64, u32, C.POINTER(u8), u32, u32, u32]),
    "rn_wire_decode_wqe_inline": (i32, [C.POINTER(u8), C.POINTER(u64)]),
    "rn_wire_build_sg_wqe": (None, [C.POINTER(u8), u32, u32, u32, C.POINTER(RnSge), i32, u64, u32, u32, u32]),
    "rn_wire_decode_wqe_sg": (i32, [C.POINTER(u8), C.POINTER(u64)]),
    "rn_k_atomic_stream": (i32, [u64, C.POINTER(u64), u32, u32, u32, u64, u32, u64, u64, u32, u64, u64, u64, u32, u32, u32, u32, u64, u64]),
    "rn_k_put_signal": (i32, [u64, u64, u64, u32, u64, u32, u32, u64, u32, u64, u32, u64, u32, u32, u64, u32, u32, u64, u64]),
    "rn_k_signal_wait": (i32, [u64, u64, u64, u64, u64, u64, u64, u64, u64, u64]),
    "rn_k_cq_watch": (i32, [u64, u64, u32, u64, u64, u64, u32, u64, u64, u64, u64, u64]),
    "rn_k_put_inline": (i32, [u64, C.POINTER(u64), u32, u64, u64, u32, u64, u32, u32, u64, u32, u64, u32, u64, u32, u32, u64, u32,
                              u32, u32, u32, u64, u64]),
    "rn_k_gather_stream": (i32, [u64, C.POINTER(u64), u32, u32, u64, u32, u64, u32, u64, u32, u64, u32, u32, u64, u32, u32, u32,
                                 u32, u32, u32, u64, u64]),
    "rn_k_read_records": (i32, [u64, u64, u64, u32, u64, u32, u64, u32, u32, u64, u64, u32, u32, u32, u64, u64]),
    "rn_gpu_page_size": (u64, []),
    "rn_dmabuf_export": (i32, [u64, u64, C.POINTER(i32)]),
    "rn_dmabuf_close": (i32, [i32]),
    "rn_dmabuf_size": (C.c_int64, [i32]),
    "rn_alloc_range": (i32, [u64, C.POINTER(u64), C.POINTER(u64)]),
    "rn_device_caps": (i32, [i32]),
    "rn_device_pci": (i32, [i32, C.c_char_p, i32]),
    "rn_p2p_open": (vp, []),
    "rn_p2p_close": (i32, [vp]),
    "rn_p2p_is_gpu_address": (i32, [vp, u64]),
    "rn_p2p_get_page_size": (i32, [vp, u64, u64, C.POINTER(u64)]),
    "rn_p2p_get_pages": (i32, [vp, u64, u64, C.POINTER(u64), C.POINTER(u32), C.POINTER(u32)]),
    "rn_p2p_put_pages": (i32, [vp, u64, u64]),
    "rn_p2p_live_pins": (i32, [vp]),
    "rn_p2p_pin_size": (C.c_int64, [vp, u64]),
    "rn_p2p_mmap": (i32, [vp, u64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "rn_p2p_window_kind": (i32, [vp, u64]),
    "rn_p2p_peek": (i32, [vp, u64, vp, u64]),
    "rn_p2p_poke": (i32, [vp, u64, vp, u64]),
    "rn_k_fill_random": (i32, [u64, u64, u64, u64]),
    "rn_k_fill_bf16": (i32, [u64, u64, u64, u64, C.c_float]),
    "rn_k_checksum": (i32, [u64, u64, u64, u64]),
    "rn_k_compare": (i32, [u64, u64, u64, u64, u64]),
    "rn_k_l2_flush": (i32, [u64, u64, u64, u32]),
    # ---- ConnectX backend (csrc/verbs/verbs_dl.cc): libibverbs / mlx5dv through dlopen
    "rn_buffer_id": (i32, [u64, C.POINTER(u64)]),
    "rn_hca_sweep_revoked": (i32, [vp]),
    "rn_mr_driver_revoked": (i32, [vp, u32]),
    "rn_qp_adopt": (i32, [vp, C.POINTER(RnGpuQp), C.POINTER(vp)]),
    "rn_qp_is_adopted": (i32, [vp]),
    "rn_verbs_compiled": (i32, []),
    "rn_verbs_why": (C.c_char_p, []),
    "rn_verbs_is_mock": (i32, []),
    "rn_verbs_libdir": (C.c_char_p, []),
    "rn_verbs_available": (i32, []),
    "rn_verbs_device_name": (i32, [i32, C.c_char_p, i32]),
    "rn_verbs_open": (vp, [C.c_char_p, i32, i32, i32]),
    "rn_verbs_close": (i32, [vp]),
    "rn_verbs_dev_name": (C.c_char_p, [vp]),
    "rn_verbs_port_active": (i32, [vp]),
    "rn_verbs_link_layer": (i32, [vp]),
    "rn_verbs_max_msg": (u32, [vp]),
    "rn_verbs_local_addr": (i32, [vp, C.POINTER(u16), C.POINTER(u8)]),
    "rn_verbs_reg_mr": (vp, [vp, u64, u64, i32, i32, u64, u32, C.POINTER(u32), C.POINTER(u32)]),
    "rn_verbs_dereg_mr": (i32, [vp]),
    "rn_verbs_create_cq": (vp, [vp, i32]),
    "rn_verbs_destroy_cq": (i32, [vp]),
    "rn_verbs_create_qp": (vp, [vp, vp, vp, u32, u32]),
    "rn_verbs_destroy_qp": (i32, [vp]),
    "rn_verbs_qpn": (u32, [vp]),
    "rn_verbs_qp_state": (u32, [vp]),
    "rn_verbs_connect": (i32, [vp, u32, u16, C.POINTER(u8)]),
    "rn_verbs_set_state": (i32, [vp, u32]),
    "rn_verbs_post_send": (i32, [vp, u32, u64, u32, u64, u32, u32, i32, u32, C.POINTER(u64)]),
    "rn_verbs_post_recv": (i32, [vp, u64, u32, u32, C.POINTER(u64)]),
    "rn_verbs_post_atomic": (i32, [vp, u32, u64, u32, u64, u32, u64, u64, i32, C.POINTER(u64)]),
    "rn_verbs_post_inline": (i32, [vp, u32, u64, u32, vp, u32, i32, u32, C.POINTER(u64)]),
    "rn_verbs_qp_max_inline": (u32, [vp]),
    "rn_verbs_post_sg": (i32, [vp, u32, C.POINTER(RnSge), i32, u64, u32, i32, u32, C.POINTER(u64)]),
    "rn_verbs_qp_max_sge": (u32, [vp]),
    "rn_verbs_poll": (i32, [vp, i32, C.POINTER(RnVWc)]),
    "rn_verbs_host_stream": (i32, [vp, u32, u64, u32, u64, u32, u32, u32, u32, u64, u32, u64, C.POINTER(u64), C.POINTER(u32)]),
    "rn_verbs_host_staged_stream": (i32, [vp, u64, u64, u64, u32, u64, u32, u32, u32, u64, u32, u64, C.POINTER(u64)]),
    "rn_verbs_raw_qp": (i32, [vp, C.POINTER(RnRawQp)]),
    "rn_verbs_db_proxy_attach": (i32, [vp, C.POINTER(u64)]),
    "rn_verbs_db_proxy_forwarded": (u64, [vp]),
    "rn_verbs_map_qp_to_gpu": (i32, [vp, C.POINTER(RnGpuQp)]),
    "rn_verbs_mock_qp_stats": (i32, [vp, C.POINTER(RnMockQpStats)]),
    "rn_verbs_mock_declare_gpu_range": (i32, [u64, u64]),
    "rn_verbs_mock_gpu_free": (i32, [u64]),
    "rn_verbs_mock_set_rnr_timeout_ms": (i32, [u64]),
    "rn_verbs_mock_post_wqe": (i32, [vp, C.POINTER(u8), C.POINTER(u64)]),
    "rn_verbs_mock_bridge_status": (C.c_char_p, []),
}

# Symbols that later build stages add; bound when present so partial builds import.
_OPTIONAL_SIGS: dict = {}


def register_optional(name, restype, argtypes):
    _OPTIONAL_SIGS[name] = (restype, argtypes)
    if _LIB is not None:
        _bind(_LIB, name, restype, argtypes, optional=True)


def _bind(lib, name, restype, argtypes, optional=False):
    try:
        fn = getattr(lib, name)
    except AttributeError:
        if optional:
            return
        raise NativeError(f"{_LIB_PATH} lacks symbol {name}; rebuild with `python -m rocnrdma_b200.build --force`")
    fn.restype = restype
    fn.argtypes = argtypes


def lib_path() -> Path:
    return _LIB_PATH


def mock_verbs_dir() -> Path:
    """Directory of the in-tree mock rdma-core provider (libibverbs.so.1 / libmlx5.so.1 look-alikes)."""
    return _LIB_PATH.parent / "mock"


def use_mock_verbs():
    """Point the ConnectX backend at the mock provider.  Must run before the backend is first used in this
    process (the libraries are dlopen()ed once); an explicit ROCNRDMA_VERBS_LIBDIR wins."""
    os.environ.setdefault("ROCNRDMA_VERBS_LIBDIR", str(mock_verbs_dir()))


def available() -> bool:
    return _LIB_PATH.exists()


def load():
    """Load (building if needed) the native library and return the ctypes handle."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if os.environ.get("ROCNRDMA_NO_AUTOBUILD"):
        if not _LIB_PATH.exists():
            raise NativeError(f"{_LIB_PATH} not built; run `python -m rocnrdma_b200.build`")
    else:
        # build() is a content-hash check when the library is current (milliseconds); a library older than its
        # sources is rebuilt rather than silently used (an edited kernel that is not the one running is the
        # worst kind of test result).
        try:
            from . import build as _build
            _build.build()
        except Exception as e:
            if not _LIB_PATH.exists():
                raise NativeError(f"{_LIB_PATH} is missing and could not be built: {e}") from e
            import warnings
            warnings.warn(f"rocnrdma_b200: could not verify that {_LIB_PATH.name} is current ({e}); using it as is", RuntimeWarning)
    # NOTE: do not set CUDA_MODULE_LOADING=EAGER here.  It would make the driver load every
    # kernel of every library in the process (torch ships GBs of them) -- minutes on a cold
    # box.  rn_hca_open preloads *our* kernels explicitly instead.
    lib = C.CDLL(str(_LIB_PATH), mode=C.RTLD_GLOBAL)
    for name, (res, args) in _SIGS.items():
        _bind(lib, name, res, args)
    for name, (res, args) in _OPTIONAL_SIGS.items():
        _bind(lib, name, res, args, optional=True)
    _LIB = lib
    return lib


def byte_count(n, what: str = "nbytes") -> int:
    """``n`` as the 32-bit byte count the native entry points take: ``ValueError`` outside ``[0, 2**32)``, where ctypes
    would silently wrap it to a shorter length.  (What fits but exceeds the maximum message length fails on the wire.)"""
    n = int(n)
    if not 0 <= n < 1 << 32:
        raise ValueError(f"{what}={n}: a byte count must lie in [0, 2**32)")
    return n


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().rn_last_error().decode(errors="replace")
        raise NativeError(f"{what or 'native call'} failed (rc={rc}): {msg}")
    return rc
