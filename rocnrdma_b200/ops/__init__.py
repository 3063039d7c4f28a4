"""Python entry points for the sm_90a kernels (K1-K6 of SURVEY.md section 2.3)."""
from .rdma import shared_post_stress, recv_consume, parse_recv, rdma_stream, StreamResult, fill_random, fill_bf16, checksum, compare, l2_flush  # noqa: F401
from .rdma import atomic_stream, put_signal, put_inline, signal_wait, parse_signal_wait, cq_watch, parse_cq_watch  # noqa: F401
from .rdma import write_read, gather_stream, read_records, parse_read_records, recv_consume_qps  # noqa: F401
from .pack import (pack_fp8_write, unpack_fp8, ref_pack_fp8, ref_unpack_fp8, record_bytes, staging_bytes,  # noqa: F401
                   PackResult, reduce_fp8, ref_reduce_fp8, parse_reduce, ReduceResult, parse_unpack, ref_allreduce_fp8,
                   relay_records, parse_relay, ref_allgather_fp8, ref_reduce_scatter_fp8, pack_fp8_scatter,
                   parse_scatter, ref_alltoall_fp8)
from .launch import result_offset  # noqa: F401
from .gemm import gemm_send, GemmResult, panel_record_bytes, ref_fp8_panels, dequant_fp8_panels  # noqa: F401
from .gemm import gemm_reduce_send, ReduceSendResult, parse_reduce_send  # noqa: F401
from .gemm_mx import gemm_mxfp8, MxOperand, MxResult, quantize_mx, dequantize_mx, ref_gemm_mxfp8  # noqa: F401
