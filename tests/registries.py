"""Save and restore pysteps' method registries around code that calls ``pysteps_b200.register()``.

``register(override=True)`` binds pysteps' stock names to this package's callables, and any
``register()`` adds the ``_b200`` names.  A test that leaves them so changes what every later test in
the process gets from pysteps' ``get_method``.  ``restored()`` snapshots all six registries and puts
back exactly what was there, whichever of them the code inside changed.  The reference must already
be importable (see golden/_refimport.py)."""
import contextlib
import importlib

# category of pysteps_b200.interface.methods() -> (pysteps module, registry attribute)
REGISTRIES = {
    "extrapolation": ("pysteps.extrapolation.interface", "_extrapolation_methods"),
    "motion": ("pysteps.motion.interface", "_methods"),
    "noise": ("pysteps.noise.interface", "_noise_methods"),
    "nowcasts": ("pysteps.nowcasts.interface", "_nowcast_methods"),
    "ensemblestats": ("pysteps.postprocessing.interface", "_ensemblestats_methods"),
    "blending": ("pysteps.blending.interface", "_blending_methods"),
}


@contextlib.contextmanager
def restored():
    """Yield {category: pysteps' registry dict}; on exit, every registry holds its entries from entry."""
    registries = {category: getattr(importlib.import_module(module), attr)
                  for category, (module, attr) in REGISTRIES.items()}
    saved = {category: dict(registry) for category, registry in registries.items()}
    try:
        yield registries
    finally:
        for category, registry in registries.items():
            registry.clear()
            registry.update(saved[category])
