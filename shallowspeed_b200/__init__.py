"""shallowspeed_b200 - an H100-native data + pipeline parallel MLP trainer with the
capabilities of siboehm/ShallowSpeed (see SURVEY.md / DESIGN.md)."""
__version__ = "0.1.0"


def _apply_tuning():
    """Export the validated kernel-variant switches of ``tuning.json`` as environment defaults (the native runtime reads
    environment variables when it builds a plan).  Explicit environment settings win; a missing / broken file is ignored."""
    import json
    import os

    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tuning.json")
    try:
        with open(path) as f:
            cfg = json.load(f)
    except (OSError, ValueError):
        return {}
    applied = {}
    for key, val in cfg.items():
        if key.startswith("SSB_") and val not in (False, None, 0, "0", ""):
            applied[key] = os.environ.setdefault(key, "1" if val is True else str(val))
    return applied


TUNING = _apply_tuning()

from . import dataset, functional, layers, optimizer, pipe, utils  # noqa: F401
