"""`openea` — drop-in import name of the reference package, served by the CUDA engine.

Every `openea.<x>` module is the SAME module object as `openea_b200.<x>`, so run/main_from_args.py and user
code written against nju-websoft/OpenEA import unchanged.
"""
import importlib
import pkgutil
import sys

import openea_b200

__version__ = '0.1-b200'
__title__ = 'openea'

_SKIP = ("openea_b200.csrc", "openea_b200._lib", "openea_b200.build")
for _m in pkgutil.walk_packages(openea_b200.__path__, "openea_b200."):
    if _m.name.startswith(_SKIP):
        continue
    _mod = importlib.import_module(_m.name)
    sys.modules["openea." + _m.name[len("openea_b200."):]] = _mod

from openea_b200 import modules, models, approaches  # noqa: E402,F401
