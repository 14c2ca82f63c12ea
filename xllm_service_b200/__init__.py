"""xllm_service_b200 — H100-native request-ingest + prefix-cache routing path.

The product is ``libxllm_ingest.so`` (CUDA sm_90a kernels behind the C-ABI of
``include/xllm_ingest.h``).  This package is the thin Python host-side mirror of
the reference's operator interfaces for that path (``Tokenizer.encode``,
``xxh3_128bits_hash``, ``GlobalKVCacheMgr.match``, ``CacheAwareRouting``) used by
the parity tests and ``bench.py``.  It contains no CPU implementation of the
path: every compute call goes through the C-ABI and fails loudly if the CUDA
library or a CUDA device is missing.
"""
from ._lib import IngestError, lib, lib_path  # noqa: F401
from .ingest import HostBuffer, Ingest  # noqa: F401

__all__ = ["HostBuffer", "Ingest", "IngestError", "lib", "lib_path"]
