"""``misc.criterion`` of the reference, served by the sm_90a implementation."""
from p2pvg_b200.misc.criterion import KLCriterion  # noqa: F401
