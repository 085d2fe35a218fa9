"""cozo_b200 — H100-native (sm_90a) HNSW k-NN search and FixedRule graph algorithms
behind CozoDB's operator surface.  See DESIGN.md / INTEGRATION.md."""
__version__ = "0.1.0"
