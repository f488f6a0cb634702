"""stract_b200 -- H100-native (sm_90a) replacements for Stract's two data-parallel ranking hot
paths, behind a C ABI (include/stract_b200.h, libstract_b200.so) and a host-side mirror of the
reference's interfaces:

  stract_b200.webgraph   Webgraph / HarmonicCentrality   (crates/core/src/webgraph/centrality/harmonic.rs)
  stract_b200.bm25       Bm25Weight / TopDocs / SignalComputer subset (crates/tantivy/src/query, crates/core/src/ranking)

The compute always runs in the CUDA library; there is no CPU fallback (the CPU restatement in
oracle/ is test infrastructure and is never imported from here).
"""
from ._lib import lib, Sb200Error, kernel_launch_count, version  # noqa: F401
