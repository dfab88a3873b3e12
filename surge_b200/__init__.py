"""surge_b200 — H100-native batched event-replay engine behind Surge's state-store boundary.

Only what the hot path needs lives here:
  csrc/        hand-written sm_90a CUDA kernels + the C ABI (include/sgr.h) -> lib/libsgr.so
  native.py    ctypes binding of the C ABI (fails loudly when the CUDA library is missing)
  formats.py   packed record / state layouts (the binary SurgeAggregateFormatting)
  programs.py  declarative fold programs for the reference's sample models
  dsl.py       text front-end that compiles a state layout + event blocks to a fold program
  engine.py    ReplayEngine: Pythonic wrapper over one sgr_engine
  ingest.py    Kafka RecordBatch bytes -> packed records (native decode) + per-partition offsets for the lag gate
  store.py     host-side mirror of the reference's plugin / state-store interfaces
  dist.py      multi-GPU rendezvous helpers (NCCL id, CUDA IPC handles) and numpy mirrors of the routing tables
  partitioner.py  KafkaPartitionProvider mirror
  synth.py     deterministic generators for the BASELINE.json configs
"""
from .native import SgrError, load_library  # noqa: F401
from .engine import ReplayEngine  # noqa: F401

__all__ = ["ReplayEngine", "SgrError", "load_library"]
