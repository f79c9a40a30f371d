"""nisqa_b200 - H100-native NISQA predict engine.

Only what the hot path needs: ``csrc/`` (sm_90a CUDA kernels + the C-ABI of
``libnisqa_b200.so``), the ctypes binding (``engine``), the host-side mirror of the reference's
predict interface (``NISQA_lib``, ``NISQA_model``), wav ingest (``wav``), rank sharding
(``dist``) and the synthetic-clip generator used by tests and ``bench.py`` (``synth``).
"""
__version__ = "0.1.0"
