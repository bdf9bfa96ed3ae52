"""oceanbase_b200 -- H100-native columnar-scan path for OceanBase micro-blocks.

Host-side Python mirror of the C-ABI in include/obgpu_scan.h. The compute path is the CUDA
library oceanbase_b200/csrc/libobgpu_scan.so (sm_90a); there is no CPU fallback: importing the
scan API without the built library, or using it without a CUDA device, raises.
"""
from .capi import (  # noqa: F401
    ObGpuError, lib, lib_path, OB_SUCCESS, OB_NOT_SUPPORTED, OB_BUF_NOT_ENOUGH, OB_INVALID_ARGUMENT,
    OB_INVALID_DATA, OB_ERR_SYS,
    WHITE_OP_EQ, WHITE_OP_LE, WHITE_OP_LT, WHITE_OP_GE, WHITE_OP_GT, WHITE_OP_NE, WHITE_OP_BT,
    WHITE_OP_IN, WHITE_OP_NU, WHITE_OP_NN,
    ENC_RAW, ENC_DICT, ENC_RLE, ENC_CONST, ENC_INTEGER_BASE_DIFF, ENC_STRING_DIFF, ENC_HEX_PACKING, ENC_STRING_PREFIX, ENC_COLUMN_EQUAL, ENC_COLUMN_SUBSTR, ENC_CS_INTEGER, ENC_CS_INT_DICT, ENC_CS_STRING, ENC_CS_STR_DICT,
    OBJ_INT, OBJ_INT32, OBJ_UINT64, OBJ_VARCHAR, OBJ_DATE, OBJ_TINYINT, OBJ_SMALLINT, OBJ_UINT32,
    DF_NOT_EXIST, DF_LOCK, DF_UPDATE, DF_INSERT, DF_DELETE,
    AGG_COUNT, AGG_SUM, AGG_SUM_PRODUCT, AGG_MIN, AGG_MAX,
    SK_IDX_MIN, SK_IDX_MAX, SK_IDX_NULL_COUNT, SK_IDX_SUM,
    BOOL_MASK_UNCERTAIN, BOOL_MASK_ALWAYS_TRUE, BOOL_MASK_ALWAYS_FALSE,
)
from .sstable import (  # noqa: F401
    Column, TableImage, encode_table, encode_block, agg_row_write, block_agg_row, table_agg_rows,
)
from .scan import (  # noqa: F401
    White, And, Or, ScanContext, PageBatch, ScanResult, CGBitmap, GroupAccumulator, flatten_filter, DATUM_DTYPE, DATUM_NULL_BIT,
)
