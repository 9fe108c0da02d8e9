"""Drop-in `source` package: the reference's entry points (`full_eval.py:4-6`, `full_run.py:3-6` import them by module
path) re-exported from the H100 implementation.  Put this repository's root in front of the reference's on `sys.path`
(or copy this directory over the reference's `source/`) and `full_eval.py` / `full_run.py` run unchanged on
libp2s_b200.so.  Only the hot-path modules exist here; everything else of the reference's `source/` (dataset generation,
figures, downloads) is out of scope (SURVEY.md section 8)."""
