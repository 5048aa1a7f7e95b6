"""tacotron-2_b200 — H100-native compute library behind the Tacotron-2 hot paths.

The directory name is not a Python identifier; import it through ``t2_import.py`` at the repo root
(``from t2_import import t2``), which registers this package as ``tacotron2_b200``.
"""
from . import lib  # noqa: F401
from . import wavenet  # noqa: F401
from . import audio  # noqa: F401
from . import tacotron  # noqa: F401
from . import init  # noqa: F401
