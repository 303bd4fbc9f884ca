"""agrep_b200 -- the H100 scan engine behind agrep's bitap/asearch/sgrep path (see DESIGN.md).
The work is done by libagrepb200.so (CUDA, sm_90a); this package is its Python-callable boundary."""
from .api import Pattern, AgrepError, bestmatch_device, corpus_host, corpus_device, corpus_spec  # noqa: F401
