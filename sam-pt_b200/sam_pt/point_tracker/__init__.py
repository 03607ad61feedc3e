"""Point trackers on the hot path: PIPS, PIPS++ and CoTracker (north star).  The reference additionally imports RAFT,
SuperGlue, TAPIR and TapNet eagerly (sam_pt/point_tracker/__init__.py:1-7); those are out of scope."""
from .tracker import PointTracker  # noqa: F401


def __getattr__(name):
    if name == "PipsPointTracker":
        from .pips import PipsPointTracker
        return PipsPointTracker
    if name in ("PipsPlusPlus", "PipsPlusPlusPointTracker"):
        from . import pips_plus_plus
        return getattr(pips_plus_plus, name)
    if name == "CoTrackerPointTracker":
        from .cotracker import CoTrackerPointTracker
        return CoTrackerPointTracker
    if name == "SuperGluePointTracker":  # SamPt only uses it in an isinstance check (sam_pt.py:189)
        class SuperGluePointTracker:  # never instantiated here
            pass
        return SuperGluePointTracker
    raise AttributeError(name)
