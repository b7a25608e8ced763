"""Import-path compatibility shim: put ``compat/`` on ``PYTHONPATH`` and an unmodified fastfp script
(``from fastfp.fastfp import FastFp`` ...) runs on the fastfp_b200 engine. The hot-path names resolve to
``fastfp_b200``; ``initialize_pta`` (enterprise model construction) is not part of this engine."""
__version__ = "0.1.0"
