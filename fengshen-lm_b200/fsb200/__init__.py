"""fsb200 — H100-native backend for the Fengshen data-parallel pretraining step (see DESIGN.md)."""
__version__ = "0.1"
