"""nrtsearch_b200 -- H100-native query-execution engine behind nrtsearch's search path.

Only what the hot path needs: csrc/ (CUDA kernels + the C ABI of include/nrtgpu.h), the host-side
mirror of the reference's query/collector interface (search.py) and the shard description +
synthetic inputs (index.py). No CPU fallback: the CUDA extension must be built and a GPU present.
"""
from ._native import NrtGpuError, NrtGpuUnsupported  # noqa: F401
from .index import HostShard, TextField  # noqa: F401
