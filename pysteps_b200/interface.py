"""Registration into pysteps' method registries (the drop-in boundary).

pysteps has no entry-point discovery for motion / extrapolation methods; the
"plugin API" is the module-level dict read by ``get_method``:
  pysteps/extrapolation/interface.py:107-111  ``_extrapolation_methods``
  pysteps/motion/interface.py:36-46           ``_methods``
  pysteps/noise/interface.py:24-45            ``_noise_methods``  ("bps": the velocity perturbator)
  pysteps/nowcasts/interface.py:44-54         ``_nowcast_methods`` ("probability": the local
                                              Lagrangian probability nowcast)
  pysteps/postprocessing/interface.py:29-33   ``_ensemblestats_methods`` ("mean", "excprob",
                                              "banddepth")
  pysteps/blending/interface.py:20-24         ``_blending_methods`` ("linear_blending",
                                              "salient_blending")
The nowcasts "extrapolation" / "lagrangian" (the extrapolation nowcast) also go into
``_nowcast_methods``.
``register()`` inserts the B200 callables under new names and, on request,
under the stock names so that ``nowcasts.steps`` (which fetches the
extrapolator by name at pysteps/nowcasts/steps.py:656 and
pysteps/nowcasts/utils.py:359) runs unchanged.
"""


def methods():
    """name -> callable for everything this package provides."""
    from .extrapolation import semilagrangian

    from .noise import motion as bps
    from .blending import interface as blending
    from .nowcasts import extrapolation as extrapolation_nowcast
    from .nowcasts import lagrangian_probability
    from .postprocessing import ensemblestats

    out = {"extrapolation": {"semilagrangian_b200": semilagrangian.extrapolate}, "motion": {},
           "noise": {"bps_b200": (bps.initialize_bps, bps.generate_bps)},
           "nowcasts": {"lagrangian_probability_b200": lagrangian_probability.forecast,
                        "probability_b200": lagrangian_probability.forecast},
           "ensemblestats": {"mean_b200": ensemblestats.mean, "excprob_b200": ensemblestats.excprob,
                             "banddepth_b200": ensemblestats.banddepth},
           # kept apart from "nowcasts" so that that entry still lists the probability models only
           "extrapolation_nowcasts": {"extrapolation_b200": extrapolation_nowcast.forecast,
                                      "lagrangian_b200": extrapolation_nowcast.forecast},
           "blending": {"linear_blending_b200": blending.get_method("linear_blending"),
                        "salient_blending_b200": blending.get_method("salient_blending")}}
    try:
        from .motion import lucaskanade
        out["motion"]["lk_b200"] = lucaskanade.dense_lucaskanade
        out["motion"]["lucaskanade_b200"] = lucaskanade.dense_lucaskanade
    except ImportError:
        pass
    try:
        from .motion import vet
        out["motion"]["vet_b200"] = vet.vet
    except ImportError:
        pass
    from .motion import proesmans
    out["motion"]["proesmans_b200"] = proesmans.proesmans
    from .motion import constant
    out["motion"]["constant_b200"] = constant.constant
    from .motion import darts
    out["motion"]["darts_b200"] = darts.DARTS
    return out


def register(override=False):
    """Insert the B200 methods into an importable ``pysteps``.

    override=False: only the ``*_b200`` names are added (the identity checks of
    pysteps/tests/test_interfaces.py keep passing).  override=True additionally
    replaces ``"semilagrangian"``, ``"lk"``/``"lucaskanade"``, ``"vet"``, ``"proesmans"``,
    ``"constant"``, ``"darts"``, the noise method ``"bps"``, the nowcasts ``"probability"`` /
    ``"lagrangian_probability"``, ``"extrapolation"`` / ``"lagrangian"``, the ensemble statistics
    ``"mean"``, ``"excprob"`` and ``"banddepth"``, and the blending methods ``"linear_blending"`` and
    ``"salient_blending"``.  Only the registries change: ``from pysteps.postprocessing.ensemblestats import
    excprob`` (and every other direct import) still gives the stock function.
    Returns the list of registered names.
    """
    import pysteps.extrapolation.interface as ei
    import pysteps.motion.interface as mi
    import pysteps.noise.interface as ni
    import pysteps.nowcasts.interface as nci
    import pysteps.blending.interface as bi
    import pysteps.postprocessing.interface as ppi

    done = []
    m = methods()
    for name, fn in m["extrapolation"].items():
        ei._extrapolation_methods[name] = fn
        done.append("extrapolation:" + name)
        if override:
            ei._extrapolation_methods[name.replace("_b200", "")] = fn
            done.append("extrapolation:" + name.replace("_b200", ""))
    for name, fn in m["motion"].items():
        mi._methods[name] = fn
        done.append("motion:" + name)
        if override:
            mi._methods[name.replace("_b200", "")] = fn
            done.append("motion:" + name.replace("_b200", ""))
    for name, fns in m["noise"].items():
        ni._noise_methods[name] = fns
        done.append("noise:" + name)
        if override:
            ni._noise_methods[name.replace("_b200", "")] = fns
            done.append("noise:" + name.replace("_b200", ""))
    for name, fn in list(m["nowcasts"].items()) + list(m["extrapolation_nowcasts"].items()):
        nci._nowcast_methods[name] = fn
        done.append("nowcasts:" + name)
        if override:
            nci._nowcast_methods[name.replace("_b200", "")] = fn
            done.append("nowcasts:" + name.replace("_b200", ""))
    for name, fn in m["ensemblestats"].items():
        ppi._ensemblestats_methods[name] = fn
        done.append("ensemblestats:" + name)
        if override:
            ppi._ensemblestats_methods[name.replace("_b200", "")] = fn
            done.append("ensemblestats:" + name.replace("_b200", ""))
    for name, fn in m["blending"].items():
        bi._blending_methods[name] = fn
        done.append("blending:" + name)
        if override:
            bi._blending_methods[name.replace("_b200", "")] = fn
            done.append("blending:" + name.replace("_b200", ""))
    return done
