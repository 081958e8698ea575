"""tuplex_b200 — an H100-native executor for Tuplex's normal-case row pipeline.

Drop-in surface: `Context.parallelize/csv -> map/filter/withColumn/mapColumn/selectColumns ->
aggregate/aggregateByKey -> collect` (tuplex/python/tuplex/{context,dataset}.py), executed by hand-written
sm_90a CUDA kernels behind the C ABI in include/tplx_gpu.h. See DESIGN.md.
"""
from .context import Context  # noqa: F401
from .dataset import DataSet  # noqa: F401

__all__ = ["Context", "DataSet"]
__version__ = "0.1.0"
