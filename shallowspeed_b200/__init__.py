"""shallowspeed_b200 - an H100-native data + pipeline parallel MLP trainer with the
capabilities of siboehm/ShallowSpeed (see SURVEY.md / DESIGN.md)."""
__version__ = "0.1.0"

from . import dataset, functional, layers, optimizer, pipe, utils  # noqa: F401
