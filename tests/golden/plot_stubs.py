"""A matplotlib stand-in for the golden generators: the reference's predict.py imports eval.py -> utils/draw_utils.py
-> matplotlib for drawing helpers the generators never call.  A meta-path finder resolves `matplotlib` and all its
submodules to permissive packages whose every attribute is a callable stand-in.  No test imports it."""
import importlib.machinery
import sys
import types


class _PermissiveModule(types.ModuleType):
    """A stand-in package whose every attribute is a callable no-op stand-in (and a package again)."""
    __path__ = []

    def __getattr__(self, name):
        if name.startswith('__'):
            raise AttributeError(name)
        return _PermissiveModule(f'{self.__name__}.{name}')

    def __call__(self, *a, **k):
        return _PermissiveModule(f'{self.__name__}()')


class _StubFinder:
    """Meta-path finder that resolves `prefix` and all its submodules to permissive stand-ins."""

    def __init__(self, prefix):
        self.prefix = prefix

    def find_spec(self, name, path=None, target=None):
        if name == self.prefix or name.startswith(self.prefix + '.'):
            return importlib.machinery.ModuleSpec(name, self, is_package=True)
        return None

    def create_module(self, spec):
        return _PermissiveModule(spec.name)

    def exec_module(self, module):
        pass


def install(prefix='matplotlib'):
    if not any(isinstance(f, _StubFinder) and f.prefix == prefix for f in sys.meta_path):
        for k in [k for k in sys.modules if k == prefix or k.startswith(prefix + '.')]:
            del sys.modules[k]
        sys.meta_path.insert(0, _StubFinder(prefix))
