"""hetu-galvatron_b200: H100-native hot path behind Hetu-Galvatron's per-layer strategy API.

Import as ``hetu_galvatron_b200`` (alias package at the repo root).  ``core`` mirrors the public names of
``galvatron.core`` (``galvatron/core/__init__.py:1-17``) for the one path this repo replaces: the
collectives every wrapped transformer layer issues under its own (PP, TP/SP, CP, DP-type, CKPT) strategy.
"""
__version__ = "0.1.0"
