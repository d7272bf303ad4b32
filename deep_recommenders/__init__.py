"""Import alias: ``deep_recommenders.*`` resolves to ``deep_recommenders_b200.*`` so the reference's
own import lines (``from deep_recommenders.keras.models.ranking import DeepFM`` ...) work
unchanged against the CUDA-native implementation."""
import importlib
import importlib.abc
import importlib.util
import sys

_TARGET = "deep_recommenders_b200"


class _AliasFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, fullname, path=None, target=None):
        if fullname == __name__ or not fullname.startswith(__name__ + "."):
            return None
        real = _TARGET + fullname[len(__name__):]
        if importlib.util.find_spec(real) is None:
            return None
        return importlib.util.spec_from_loader(fullname, self)

    def create_module(self, spec):
        real = _TARGET + spec.name[len(__name__):]
        return importlib.import_module(real)

    def exec_module(self, module):
        pass


sys.meta_path.insert(0, _AliasFinder())
_real = importlib.import_module(_TARGET)
__version__ = _real.__version__
__path__ = []  # submodules come from the alias finder
