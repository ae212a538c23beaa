"""Drop-in alias: put `compat/` FIRST on PYTHONPATH and the reference's `train_dna_qwen.py` / `reason.py` import the
CUDA hot path under the reference's own module names (only the hot-path symbols are provided; the reference's
CPU-side packages -- dataset, dna_modules, processor -- stay the reference's, see INTEGRATION.md)."""
