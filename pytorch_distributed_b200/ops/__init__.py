"""Hand-written sm_90a ops with PyTorch reference fall-backs (CPU / oracle)."""
