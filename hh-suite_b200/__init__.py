"""hh-suite_b200: GPU-native (H100) Viterbi HMM-HMM alignment + cs219 prefilter behind the HH-suite3 call
boundary.  The product is the C-ABI library (include/hhg.h, csrc/); this package is its thin host
mirror in Python (ctypes) plus the synthetic-data generator used by tests and bench.py."""
from . import build, capi, ffindex, mac, pipeline, prefilter, runner, shard, synth  # noqa: F401
from .capi import Comm, Context, CsDB, HhgError, HostStore, Plan, RecordSource, StagedDB, TargetDB, viterbi_search, expand_path  # noqa: F401
