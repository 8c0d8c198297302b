"""Install ppq_b200 into an unmodified OpenPPL/ppq checkout (drop-in boundary, SURVEY.md §8b).

    import ppq, ppq_b200.install
    ppq_b200.install.install()            # CUDA_COMPLIER now serves the sm_90a extension; complie() is a no-op
    with ppq.api.ENABLE_CUDA_KERNEL(): ...

Everything ppq.core.ffi.CUDA calls (`CUDA_COMPLIER.CUDA_EXTENSION.<name>(...)`, /root/reference/ppq/core/ffi.py:78-344)
lands in ppq_b200/_C.so, which exports the same 20 names with the same positional signatures.

`replace_observers=True` additionally swaps the range observers for the device-resident ones of ppq_b200.observer.  The reference
decides which observers need a second calibration pass by EXACT TYPE (`type(var_observer) not in {TorchHistObserver,
TorchMSEObserver}`, ppq/quantization/optim/calibration.py:195 and optim/ssd.py:445), so the class names those modules
imported are rebound as well -- otherwise a replaced 'kl' observer would be dropped after phase 1 and its config would stay
INITIAL (tests/test_gpu_graph_parity.py drives the reference's own RuntimeCalibrationPass through this).
"""

_saved = {}
_SWAPPED = ('minmax', 'kl', 'mse', 'percentile')
# (module, attribute) pairs of the reference that hold observer classes by name and compare against them with type(...)
_TYPE_CHECK_SITES = (('ppq.quantization.optim.calibration', 'TorchHistObserver'), ('ppq.quantization.optim.calibration', 'TorchMSEObserver'),
                     ('ppq.quantization.optim.calibration', 'TorchMinMaxObserver'), ('ppq.quantization.optim.ssd', 'TorchHistObserver'))


def install(replace_observers: bool = True):
    """Route ppq.core.ffi.CUDA to the sm_90a extension; with replace_observers also swap the 'minmax' / 'kl' / 'mse' / 'percentile'
    observers for the device-resident ones (they need CUDA tensors: a CPU-path calibration of the real PPQ should call uninstall()
    first or pass False)."""
    import importlib

    import ppq.core.ffi as ref_ffi
    from .ffi import extension
    ext = extension()
    helper = ref_ffi.CUDA_COMPLIER
    if 'complie' not in _saved:
        _saved['extension'] = getattr(helper, '__CUDA_EXTENTION__', None)
        _saved['complie'] = type(helper).complie
    helper.__CUDA_EXTENTION__ = ext                      # attribute name ends with "__": no name mangling (ffi.py:19)
    type(helper).complie = lambda self: None             # ENABLE_CUDA_KERNEL.__init__ always calls complie() (api/interface.py:925-927)
    if replace_observers:
        import ppq.quantization.observer as ref_obs
        from . import observer as obs
        _saved.setdefault('observers', {k: ref_obs.OBSERVER_TABLE[k] for k in _SWAPPED})
        for k in _SWAPPED:
            ref_obs.OBSERVER_TABLE[k] = obs.OBSERVER_TABLE[k]
        sites = _saved.setdefault('type_sites', {})
        for mod_name, attr in _TYPE_CHECK_SITES:
            try:
                mod = importlib.import_module(mod_name)
            except Exception:                                # an optional pass that does not import in this environment
                continue
            if hasattr(mod, attr):
                sites.setdefault((mod_name, attr), getattr(mod, attr))
                setattr(mod, attr, getattr(obs, attr))
    return ext


def uninstall():
    """Undo install(): the reference's own JIT helper, extension slot and observers are back in place."""
    if not _saved: return
    import importlib

    import ppq.core.ffi as ref_ffi
    helper = ref_ffi.CUDA_COMPLIER
    helper.__CUDA_EXTENTION__ = _saved.pop('extension')
    type(helper).complie = _saved.pop('complie')
    obs = _saved.pop('observers', None)
    if obs:
        import ppq.quantization.observer as ref_obs
        ref_obs.OBSERVER_TABLE.update(obs)
    for (mod_name, attr), cls in _saved.pop('type_sites', {}).items():
        setattr(importlib.import_module(mod_name), attr, cls)
