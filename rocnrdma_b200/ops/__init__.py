"""Python entry points for the sm_90a kernels (K1-K6 of SURVEY.md section 2.3)."""
from .rdma import shared_post_stress, recv_consume, parse_recv, rdma_stream, StreamResult, fill_random, fill_bf16, checksum, compare, l2_flush  # noqa: F401
from .pack import (pack_fp8_write, unpack_fp8, ref_pack_fp8, ref_unpack_fp8, record_bytes, staging_bytes,  # noqa: F401
                   PackResult)
from .gemm import gemm_send, GemmResult, panel_record_bytes, ref_fp8_panels, dequant_fp8_panels  # noqa: F401
from .gemm_mx import gemm_mxfp8, MxOperand, MxResult, quantize_mx, dequantize_mx  # noqa: F401
