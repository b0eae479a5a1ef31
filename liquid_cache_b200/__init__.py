"""liquid_cache_b200 — the insert / get / eval_predicate hot path of XiangpengHao/liquid-cache,
rebuilt as sm_90a CUDA kernels over HBM-resident liquid columns (see DESIGN.md).

The compute lives in lib/liblc_gpu.so (C ABI: include/lc_gpu.h). Importing this package on a machine
without the built library, or calling into it without an H100, raises: there is no CPU implementation here.
"""
from . import _native
from .cache import (EntryID, EvaluatePredicate, Get, GpuLiquidArray, Insert, LiquidCache, LiquidCacheBuilder, Scan,
                    parquet_array_id, selection_bits)
from .expr import (BinaryExpr, CacheExpression, CastColumnExpr, CastExpr, Column, DynamicFilterPhysicalExpr, InListExpr,
                   LikeExpr, LiquidExpr, Literal, ScalarFunctionExpr, TryCastExpr, split_disjunction)

__all__ = [
    "EntryID", "EvaluatePredicate", "Get", "GpuLiquidArray", "Insert", "LiquidCache", "LiquidCacheBuilder", "Scan",
    "parquet_array_id", "selection_bits", "BinaryExpr", "CacheExpression", "CastColumnExpr", "CastExpr", "Column",
    "DynamicFilterPhysicalExpr", "InListExpr", "LikeExpr", "LiquidExpr", "Literal", "ScalarFunctionExpr", "TryCastExpr",
    "split_disjunction",
]
