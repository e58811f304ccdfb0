"""Library-wide constants (parity: reference pipegoose/constants.py:1-29)."""

SEED = 69

# checkpoint naming: one file per (tensor-parallel rank, pipeline-parallel rank)
CHECKPOINT_WEIGHTS_NAME = "pytorch_model_tp_{}_pp_{}.bin"
CHECKPOINT_OPTIM_NAME = "optimizer_tp_{}_pp_{}_dp_{}.bin"
CHECKPOINT_PATH_NAME = "./"

# data parallel: gradient bucket size (MB).  The fused NVLink reducer works on buckets this big.
BUCKET_SIZE_MB = 25

# pipeline parallel
WORKER_NAME = "RPC_GLOBAL_WORKER_{}"
PIPELINE_MIN_WORKERS = 1
PIPELINE_MAX_WORKERS = 1
JOB_KEY_LENGTH = 15

# H100 SXM facts used by heuristics (grid sizing, bucket sizing, layout planning) and as roofline denominators
H100_NUM_SMS = 132
H100_L2_BYTES = 50 * 1024 * 1024
H100_HBM_BYTES = 80 * 1024**3
H100_BF16_DENSE_FLOPS = 989e12     # data sheet, dense bf16 at the 700 W limit (not reached)
H100_NVLINK_BYTES_PER_S = 450e9    # NVLink4: 900 GB/s bidirectional per GPU = 450 GB/s per direction (data sheet)
# the names these constants had before the port (same values), for code that imports them
B200_NUM_SMS = H100_NUM_SMS
B200_L2_BYTES = H100_L2_BYTES
B200_HBM_BYTES = H100_HBM_BYTES
MAX_NVLINK_PEERS = 8
