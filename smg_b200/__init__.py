"""smg_b200 — H100-native drop-in for SMG's `--policy cache_aware` worker pick.

The product is the C-ABI library `libsmgx.so` (hand-written sm_90a CUDA, include/smgx.h).  This package is the thin
host-side mirror of the reference's plugin surface (policies::CacheAwarePolicy, kv_index::PositionalIndexer) used by
the parity tests and bench.py; it adds no logic of its own and has no CPU fallback.
"""
from .policy import (BasicWorker, CacheAwareConfig, CacheAwarePolicy, KvEventMonitor, PositionalIndexer, SelectWorkerInfo,  # noqa: F401
                     PolicyFactory, TiktokenTokenizer, HuggingFaceTokenizer, TokenTree, Tree, HashRing, PrefixHashConfig, PrefixHashPolicy, PowerOfTwoPolicy,
                     ConsistentHashingPolicy)
from ._lib import SmgxError  # noqa: F401
