"""Drop-in import name: ``import ahocorasick_rs`` resolves to the CUDA build
(ahocorasick_rs_b200), so code and tests written against the reference run
unmodified."""
from ahocorasick_rs_b200 import *  # noqa: F401,F403
from ahocorasick_rs_b200 import __all__  # noqa: F401
