from .cuda_lib import lib, check, stream_ptr, PRO_RMSNORM, PRO_PLAIN, EPI_STORE, EPI_RESIDUAL, EPI_SWIGLU, EPI_ARGMAX
from .cuda_lib import GEPI_STORE_F32, GEPI_RESIDUAL, GEPI_SWIGLU_BF16
from .q40 import DeviceQ40, DeviceDense, repack_q40, gemv_q40, gemv_dense, gemm_q40_tc, gemm_q40_tc_plan, GemmPlan, rmsnorm_bf16
from .q40 import gemv_q40_plan, GemvPlan, gemv_q40_argmax, gemv_q40_argmax_rows, argmax_advance, gemv_dense_smem_bytes
