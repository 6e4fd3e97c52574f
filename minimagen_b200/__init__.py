"""minimagen_b200 -- H100-native (sm_90a) implementation of MinImagen's U-Net denoising hot path.

Drop-in module layout (same names as the reference package `minimagen`):
    minimagen_b200.Unet             Unet, Base, Super, BaseTest, SuperTest
    minimagen_b200.Imagen           Imagen
    minimagen_b200.diffusion_model  GaussianDiffusion
    minimagen_b200.layers, .helpers, .t5

`install_as_minimagen()` makes the reference's own callers (`train.py`, `inference.py`, `minimagen.generate`,
`minimagen.training`) import these modules under the reference's names (see INTEGRATION.md).
"""
import importlib
import importlib.util
import os
import sys
import types

__version__ = "0.2.0"

HOT_PATH_MODULES = ('Unet', 'Imagen', 'diffusion_model', 'layers', 'helpers', 't5')


def _find_reference(reference_root=None):
    """Directory of the reference's `minimagen` package (the one holding generate.py / training.py), or None."""
    cands = []
    if reference_root:
        cands.append(os.path.join(reference_root, 'minimagen'))
    if os.environ.get('MINIMAGEN_REFERENCE'):
        cands.append(os.path.join(os.environ['MINIMAGEN_REFERENCE'], 'minimagen'))
    mod = sys.modules.get('minimagen')
    if mod is not None and getattr(mod, '__name__', '') == 'minimagen':
        cands.extend(getattr(mod, '__path__', []))
    for p in sys.path:
        cands.append(os.path.join(p or '.', 'minimagen'))
    here = os.path.dirname(os.path.abspath(__file__))
    for c in cands:
        c = os.path.abspath(c)
        if c != here and os.path.isfile(os.path.join(c, 'generate.py')) and os.path.isfile(os.path.join(c, 'Unet.py')):
            return c
    return None


def install_as_minimagen(reference_root=None):
    """Register the hot-path modules of this package under the reference's names.

    * When the reference package is importable (already imported, on sys.path, `reference_root=` or $MINIMAGEN_REFERENCE),
      `minimagen` stays a package whose `__path__` is the reference's directory -- so `minimagen.generate` and
      `minimagen.training` are the reference's own files -- and only `minimagen.{Unet,Imagen,diffusion_model,layers,
      helpers,t5}` are replaced by this package's modules (both in sys.modules and as attributes, so
      `from minimagen import Unet` resolves here too).  Reference modules that were imported earlier and captured the
      reference's classes (`minimagen.generate`, `minimagen.training`) are dropped so that they re-import the aliases.
    * Otherwise `minimagen` becomes an alias package holding only the hot-path modules.

    Works in either order relative to `import minimagen`.  Returns the `minimagen` package module."""
    ref_dir = _find_reference(reference_root)
    pkg = types.ModuleType('minimagen')
    pkg.__package__ = 'minimagen'
    pkg.__b200__ = True
    if ref_dir is not None:
        pkg.__path__ = [ref_dir]
        pkg.__file__ = os.path.join(ref_dir, '__init__.py')
        pkg.__spec__ = importlib.util.spec_from_file_location('minimagen', pkg.__file__,
                                                              submodule_search_locations=[ref_dir])
    else:
        here = os.path.dirname(os.path.abspath(__file__))
        pkg.__path__ = [here]
        pkg.__file__ = os.path.join(here, '__init__.py')
        pkg.__spec__ = importlib.util.spec_from_file_location('minimagen', pkg.__file__,
                                                              submodule_search_locations=[here])
    for name in list(sys.modules):
        if name == 'minimagen' or name.startswith('minimagen.'):
            del sys.modules[name]
    sys.modules['minimagen'] = pkg
    for name in HOT_PATH_MODULES:
        mod = importlib.import_module(f'{__name__}.{name}')
        sys.modules[f'minimagen.{name}'] = mod
        setattr(pkg, name, mod)
    return pkg
