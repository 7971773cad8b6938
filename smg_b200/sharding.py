"""Worker-id sharding of the event-driven pick across the GPUs of one box (BASELINE config 4, SURVEY §8e).

Each rank owns a contiguous range of the global worker slice (so that "last max wins" keeps meaning "highest global
index"), indexes only its own workers' KV blocks, runs the candidate kernels on the FULL request batch, and the per-request
24-byte candidates are all-gathered and merged on every rank (smgx_shard_reduce_device).  The pick equals the reference search run
on each shard's index alone, merged in rank order; that is the whole-fleet pick when every index entry holds workers of one prefix
chain, but not in general (the jump search's count test and retain guard compare sizes of whole-fleet worker sets; DESIGN.md §4d
gives a counterexample).  torch.distributed is plumbing
here (NCCL over NVLink on a multi-GPU box, gloo when the ranks share one device); the kernels and the C ABI are the product.
"""
import ctypes as C

import numpy as np

from . import _lib
from .policy import BasicWorker, CacheAwareConfig, CacheAwarePolicy

CAND_BYTES, FLEET_BYTES = 24, 40


def shard_range(n_workers: int, rank: int, world: int):
    """Contiguous, balanced ranges in global slice order."""
    base, rem = divmod(n_workers, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class ShardedEventRouter:
    def __init__(self, urls, rank: int, world: int, config: CacheAwareConfig, jump_size: int = 64, device_id: int = 0,
                 max_batch: int = 65536, max_tokens_per_request: int = 8192):
        self.rank, self.world, self.urls = rank, world, list(urls)
        self.ranges = [shard_range(len(urls), g, world) for g in range(world)]
        self.lo, self.hi = self.ranges[rank]
        self.policy = CacheAwarePolicy(config, device_id=device_id, max_batch=max_batch, max_tokens_per_request=max_tokens_per_request)
        self.workers = [BasicWorker(u) for u in self.urls[self.lo:self.hi]]
        self.policy.init_workers(self.workers)
        self.monitor = self.policy.kv_event_monitor(config.block_size)
        self.indexer = self.monitor.create_indexer("unknown", jump_size)
        self.policy.set_kv_event_monitor(self.monitor)
        for w in self.workers:                       # local ids follow local slice order
            self.indexer.intern_worker(w.url())
        self.gbase = np.asarray([r[0] for r in self.ranges], dtype=np.uint32)
        self._max_batch = max_batch
        self._h, self._L = self.policy._h, _lib.load()

    def connect_peers(self, all_gather_bytes):
        """Peer-memory exchange (smgx_shard_exchange_*): `all_gather_bytes(np.uint8[64]) -> np.uint8[world*64]` swaps the CUDA IPC
        handles once; afterwards select_fused needs no collective and no host synchronisation between the kernels."""
        handle = np.zeros(64, np.uint8)
        self._h.call("smgx_shard_exchange_create", self.world, self.rank, self._max_batch, handle.ctypes.data_as(C.c_void_p))
        handles = np.ascontiguousarray(all_gather_bytes(handle), dtype=np.uint8)
        self._h.call("smgx_shard_exchange_connect", handles.ctypes.data_as(C.c_void_p))

    def select_fused_device(self, d_tokens, d_offsets, n: int, max_request_tokens: int, d_out, lane: int = 0):
        """Device pointers in, asynchronous on `lane`: candidates → stores into every rank's gather buffer → wait → merge."""
        self._h.call("smgx_shard_select_fused_device", self.model, lane, d_tokens, d_offsets, n, max_request_tokens,
                     self.gbase.ctypes.data_as(C.c_void_p), d_out, None)

    def select_fused(self, tokens, offsets, max_request_tokens: int):
        """Host arrays in/out around select_fused_device (tests)."""
        tokens = np.ascontiguousarray(tokens, dtype=np.uint32)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
        n = offsets.size - 1
        h, L = self._h, self._L
        err = _lib.new_err()
        alloc = lambda nbytes: L.smgx_device_alloc(h.p, max(nbytes, 16), C.byref(err))
        d_tok, d_off, d_out = alloc(tokens.nbytes), alloc(offsets.nbytes), alloc(n * 4)
        if tokens.size:
            h.call("smgx_memcpy_h2d", d_tok, tokens.ctypes.data_as(C.c_void_p), tokens.nbytes)
        h.call("smgx_memcpy_h2d", d_off, offsets.ctypes.data_as(C.c_void_p), offsets.nbytes)
        self.select_fused_device(d_tok, d_off, n, max_request_tokens, d_out)
        h.call("smgx_synchronize")
        out = np.zeros(max(n, 1), np.int32)
        h.call("smgx_memcpy_d2h", out.ctypes.data_as(C.c_void_p), d_out, n * 4)
        for d in (d_tok, d_off, d_out):
            L.smgx_device_free(h.p, d)
        return out[:n]

    def owns(self, global_idx: int) -> bool:
        return self.lo <= global_idx < self.hi

    def local_id(self, global_idx: int) -> int:
        return global_idx - self.lo

    def set_fleet_state(self, loads, healthy, circuit_ok=None):
        """Global arrays; each rank keeps its slice."""
        for k, w in enumerate(self.workers):
            g = self.lo + k
            w.set_load(int(loads[g])); w.set_healthy(bool(healthy[g]))
            w.set_circuit_ok(True if circuit_ok is None else bool(circuit_ok[g]))
        self.model = self.policy._push_fleet(self.workers)

    def select(self, tokens, offsets, max_request_tokens: int, all_gather):
        """tokens/offsets: numpy (host).  all_gather(bytes_tensor_like np.uint8 array) -> concatenated [world, ...] np.uint8.
        Returns global worker indices (−1 = None)."""
        tokens = np.ascontiguousarray(tokens, dtype=np.uint32)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
        n = offsets.size - 1
        h, L = self._h, self._L
        err = _lib.new_err()
        alloc = lambda nbytes: L.smgx_device_alloc(h.p, max(nbytes, 16), C.byref(err))
        d_tok, d_off = alloc(tokens.nbytes), alloc(offsets.nbytes)
        d_cand, d_fleet = alloc(n * CAND_BYTES), alloc(FLEET_BYTES)
        if tokens.size:
            h.call("smgx_memcpy_h2d", d_tok, tokens.ctypes.data_as(C.c_void_p), tokens.nbytes)
        h.call("smgx_memcpy_h2d", d_off, offsets.ctypes.data_as(C.c_void_p), offsets.nbytes)
        h.call("smgx_shard_candidates_device", self.model, 0, d_tok, d_off, n, max_request_tokens, d_cand, d_fleet)
        h.call("smgx_synchronize")
        cand, fleet = np.zeros(n * CAND_BYTES, np.uint8), np.zeros(FLEET_BYTES, np.uint8)
        h.call("smgx_memcpy_d2h", cand.ctypes.data_as(C.c_void_p), d_cand, cand.nbytes)
        h.call("smgx_memcpy_d2h", fleet.ctypes.data_as(C.c_void_p), d_fleet, fleet.nbytes)
        all_cand, all_fleet = all_gather(cand), all_gather(fleet)      # [world * n * 24], [world * 40]
        d_all_c, d_all_f, d_out = alloc(all_cand.nbytes), alloc(all_fleet.nbytes), alloc(n * 4)
        h.call("smgx_memcpy_h2d", d_all_c, all_cand.ctypes.data_as(C.c_void_p), all_cand.nbytes)
        h.call("smgx_memcpy_h2d", d_all_f, all_fleet.ctypes.data_as(C.c_void_p), all_fleet.nbytes)
        h.call("smgx_shard_reduce_device", 0, d_all_c, d_all_f, self.gbase.ctypes.data_as(C.c_void_p), self.world, n, d_out, None)
        h.call("smgx_synchronize")
        out = np.zeros(max(n, 1), np.int32)
        h.call("smgx_memcpy_d2h", out.ctypes.data_as(C.c_void_p), d_out, n * 4)
        for d in (d_tok, d_off, d_cand, d_fleet, d_all_c, d_all_f, d_out):
            L.smgx_device_free(h.p, d)
        return out[:n]
