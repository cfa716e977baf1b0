"""Drop-in `import MinkowskiEngine as ME` → the sm_90a engine (pasco_b200.me)."""
import os as _os, sys as _sys
_sys.path.insert(0, _os.path.dirname(_os.path.dirname(_os.path.dirname(_os.path.abspath(__file__)))))
from pasco_b200.me import *            # noqa: F401,F403
from pasco_b200.me import utils, __version__, CoordinateManager, CoordinateMapKey  # noqa: F401
