"""Registration into pysteps' method registries (the drop-in boundary).

pysteps has no entry-point discovery for these methods; the "plugin API" is the module-level dict
that each subpackage's ``get_method`` reads.  Each subpackage of this package names what it provides
in one mapping, ``PROVIDED``, from pysteps' stock name to this package's callable.  Its own registry
holds those names and the same callables under ``name + "_b200"``; ``register()`` inserts the
``_b200`` names into pysteps' registries and, on request, the stock names too, so that
``nowcasts.steps`` (which fetches the extrapolator by name at pysteps/nowcasts/steps.py:656 and
pysteps/nowcasts/utils.py:359) runs unchanged.
"""

SUFFIX = "_b200"


def with_b200_names(provided):
    """A subpackage's registry entries for ``provided``: every stock name and ``name + "_b200"``,
    bound to the same object."""
    return {key: fn for name, fn in provided.items() for key in (name, name + SUFFIX)}


def _registries():
    """(category, pysteps module, registry attribute, PROVIDED) for every registry this package
    publishes into."""
    from .blending import interface as blending
    from .extrapolation import interface as extrapolation
    from .motion import interface as motion
    from .noise import interface as noise
    from .nowcasts import interface as nowcasts
    from .postprocessing import interface as postprocessing

    return (("extrapolation", "pysteps.extrapolation.interface", "_extrapolation_methods", extrapolation.PROVIDED),
            ("motion", "pysteps.motion.interface", "_methods", motion.PROVIDED),
            ("noise", "pysteps.noise.interface", "_noise_methods", noise.PROVIDED),
            ("nowcasts", "pysteps.nowcasts.interface", "_nowcast_methods", nowcasts.PROVIDED),
            ("ensemblestats", "pysteps.postprocessing.interface", "_ensemblestats_methods", postprocessing.PROVIDED),
            ("blending", "pysteps.blending.interface", "_blending_methods", blending.PROVIDED))


def methods():
    """category -> {name + "_b200": callable} for everything this package provides."""
    return {category: {name + SUFFIX: fn for name, fn in provided.items()}
            for category, _, _, provided in _registries()}


def register(override=False):
    """Insert the B200 methods into an importable ``pysteps``.

    override=False: only the names of ``methods()`` are added (the identity checks of
    pysteps/tests/test_interfaces.py keep passing).  override=True also binds the same names
    without ``_b200``, so pysteps' stock names resolve to this package.  Only the registries change:
    ``from pysteps.postprocessing.ensemblestats import excprob`` (and every other direct import)
    still gives the stock function.
    Returns the registered names as ``"category:name"``.
    """
    import importlib

    # every pysteps registry is imported before the first one is written
    tables = [(category, getattr(importlib.import_module(module), attr), provided)
              for category, module, attr, provided in _registries()]
    done = []
    for category, registry, provided in tables:
        for name, fn in provided.items():
            registry[name + SUFFIX] = fn
            done.append(category + ":" + name + SUFFIX)
            if override:
                registry[name] = fn
                done.append(category + ":" + name)
    return done
