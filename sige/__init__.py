"""Drop-in alias of the reference package name: ``import sige`` / ``from sige.nn import ...`` /
``from sige.utils import ...`` resolve to the H100-native implementation in ``sige_b200``
(reference sige/__init__.py:1-2)."""
from sige_b200 import __version__  # noqa: F401
from . import nn, utils  # noqa: F401
