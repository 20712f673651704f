"""Install the drop-in modules under the reference's module name.

    import lama_b200.patch as p; p.install()      # BEFORE anything imports saicinpainting.training.modules
    # ... then run the reference unchanged, e.g. runpy.run_path("bin/predict.py")

``install()`` registers ``lama_b200.modules`` as ``sys.modules['saicinpainting.training.modules.ffc']``, so the
reference's own import sites bind to the replacement:

  * ``saicinpainting/training/modules/__init__.py:3``   ``from …ffc import FFCResNetGenerator``  (make_generator)
  * ``saicinpainting/training/modules/pix2pixhd.py:12`` ``from …ffc import FFCResnetBlock``
  * ``saicinpainting/evaluation/refinement.py:13``      ``from …ffc import FFCResnetBlock``      (isinstance check :271)

Ordering trap (SURVEY.md §8b): the reference's ``ffc.py`` imports ``saicinpainting.training.modules.base``,
which executes the package ``__init__`` and binds the *reference* class by name.  ``lama_b200.modules`` therefore
never imports the reference package.  If the package was already imported, ``install()`` rebinds the three
import sites instead.  ``uninstall()`` restores everything (used by the tests).

The LaMa-Regular generators (``pix2pixhd_global``) are bound too: ``GlobalGenerator`` in
``saicinpainting.training.modules.pix2pixhd`` and in the package namespace ``make_generator`` reads
(``modules/__init__.py:4,14``).  ``install()`` runs before those modules exist, so an import hook rebinds the name
right after ``pix2pixhd.py`` has run, before the package ``__init__`` copies it.  The bound class builds the drop-in
``lama_b200.pix2pixhd.GlobalGenerator``, except for the options that need reference-only classes (depthwise or
multidilated convs, ``dilation_block_kind='multi'``), for which it builds the reference's own class.
``pix2pixhd.ResnetBlock`` stays the reference's: ``multiscale.py`` builds it with options the drop-in lacks.
"""
import importlib
import importlib.abc
import importlib.machinery
import inspect
import sys

_NAME = "saicinpainting.training.modules.ffc"
_SITES = [("saicinpainting.training.modules", ["FFCResNetGenerator"]),
          ("saicinpainting.training.modules.pix2pixhd", ["FFCResnetBlock"]),
          ("saicinpainting.evaluation.refinement", ["FFCResnetBlock"])]
_P2P = "saicinpainting.training.modules.pix2pixhd"
_PKG = "saicinpainting.training.modules"
_saved = {}


def _global_generator_site(reference):
    """The class bound as ``GlobalGenerator`` at the reference's import sites: calling it builds the drop-in, or the
    ``reference`` class for options only the reference implements."""
    from .pix2pixhd import GlobalGenerator, reference_only_options
    sig = inspect.signature(GlobalGenerator.__init__)

    class _GlobalGeneratorSite(GlobalGenerator):
        def __new__(cls, *args, **kwargs):
            opts = sig.bind(None, *args, **kwargs).arguments
            if reference_only_options(**{k: v for k, v in opts.items() if k != "self"}):
                return reference(*args, **kwargs)
            return GlobalGenerator(*args, **kwargs)       # not an instance of cls: __init__ is not run again

    _GlobalGeneratorSite.reference = reference
    _GlobalGeneratorSite.__name__ = _GlobalGeneratorSite.__qualname__ = "GlobalGenerator"
    return _GlobalGeneratorSite


def _bind_global_generator(mod):
    cur = getattr(mod, "GlobalGenerator", None)
    if cur is None or hasattr(cur, "reference"):
        return
    setattr(mod, "GlobalGenerator", _global_generator_site(cur))


class _Pix2pixhdHook(importlib.abc.MetaPathFinder):
    """Rebinds ``GlobalGenerator`` as soon as the reference's ``pix2pixhd.py`` has executed."""

    def find_spec(self, fullname, path, target=None):
        if fullname != _P2P:
            return None
        spec = importlib.machinery.PathFinder.find_spec(fullname, path)
        if spec is None or spec.loader is None:
            return spec
        spec.loader = _BindingLoader(spec.loader)
        return spec


class _BindingLoader(importlib.abc.Loader):
    def __init__(self, inner):
        self.inner = inner

    def create_module(self, spec):
        return self.inner.create_module(spec)

    def exec_module(self, module):
        self.inner.exec_module(module)
        _bind_global_generator(module)


_HOOK = _Pix2pixhdHook()


def install():
    from . import modules
    if _NAME in sys.modules and sys.modules[_NAME] is modules:
        return modules
    if _HOOK not in sys.meta_path:
        sys.meta_path.insert(0, _HOOK)
    for name in (_P2P, _PKG):          # already imported: rebind now
        if name in sys.modules:
            _bind_global_generator(sys.modules[name])
    _saved.setdefault("module", sys.modules.get(_NAME))
    sys.modules[_NAME] = modules
    pkg = sys.modules.get("saicinpainting.training.modules")
    if pkg is not None:
        setattr(pkg, "ffc", modules)
    # the package (or a sibling) was imported before us: rebind the names it already copied
    for mod_name, names in _SITES:
        mod = sys.modules.get(mod_name)
        if mod is None:
            continue
        for n in names:
            if hasattr(mod, n) and getattr(mod, n) is not getattr(modules, n):
                _saved[(mod_name, n)] = getattr(mod, n)
                setattr(mod, n, getattr(modules, n))
    return modules


def uninstall():
    if _HOOK in sys.meta_path:
        sys.meta_path.remove(_HOOK)
    for name in (_P2P, _PKG):
        mod = sys.modules.get(name)
        cur = getattr(mod, "GlobalGenerator", None) if mod is not None else None
        if cur is not None and hasattr(cur, "reference"):
            setattr(mod, "GlobalGenerator", cur.reference)
    orig = _saved.pop("module", None)
    if orig is not None:
        sys.modules[_NAME] = orig
    else:
        sys.modules.pop(_NAME, None)
    for key in [k for k in _saved if isinstance(k, tuple)]:
        mod = sys.modules.get(key[0])
        if mod is not None:
            setattr(mod, key[1], _saved[key])
        _saved.pop(key)


def installed() -> bool:
    from . import modules
    return sys.modules.get(_NAME) is modules
