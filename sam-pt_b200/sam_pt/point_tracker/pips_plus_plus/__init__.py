from .pips_plus_plus import PipsPlusPlus  # noqa: F401
from .tracker import PipsPlusPlusPointTracker  # noqa: F401
