"""H100-native synthetic-PTA residual generator: a drop-in for the injection path of
bencebecsy/pta_replicator (``load_pulsar`` / ``make_ideal`` / ``add_measurement_noise`` /
``add_jitter`` / ``add_red_noise`` / ``add_gwb`` / ``add_cgw``) plus the batched engine
(``PulsarBatch``) that the reference lacks.  Importing is cheap and CPU-safe; any injection
call needs a CUDA device and the in-tree ``libptar_b200.so`` (no CPU fallback).
"""
from .simulate import (SimulatedPulsar, load_from_directories, load_pulsar, make_ideal,  # noqa: F401
                       pulsar_from_arrays, simulate_pulsar)

__all__ = ["SimulatedPulsar", "load_pulsar", "load_from_directories", "simulate_pulsar", "make_ideal",
           "pulsar_from_arrays", "add_measurement_noise", "add_jitter", "add_efac", "add_ecorr",
           "add_red_noise", "add_gwb", "add_cgw", "add_catalog_of_cws", "add_burst", "add_noise_transient",
           "add_gw_memory", "add_gwb_plus_outlier_cws", "PulsarBatch"]


def __getattr__(name):  # lazy: keeps `import pta_replicator_b200` free of torch
    if name in ("add_measurement_noise", "add_jitter", "add_efac", "add_ecorr", "quantize_fast"):
        from . import white_noise
        return getattr(white_noise, name)
    if name in ("add_red_noise", "add_gwb", "create_fourier_design_matrix_red", "add_dm_noise", "add_chromatic_noise"):
        from . import red_noise
        return getattr(red_noise, name)
    if name in ("add_cgw", "add_catalog_of_cws", "add_burst", "add_noise_transient", "add_gw_memory",
                "add_gwb_plus_outlier_cws"):
        from . import deterministic
        return getattr(deterministic, name)
    if name == "PulsarBatch":
        from .engine import PulsarBatch
        return PulsarBatch
    raise AttributeError(name)
