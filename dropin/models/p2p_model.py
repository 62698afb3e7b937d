"""models.p2p_model of the reference, served by the sm_90a implementation."""
from p2pvg_b200.models.p2p_model import *  # noqa: F401,F403
from p2pvg_b200.models import p2p_model as _impl

globals().update({k: v for k, v in vars(_impl).items() if not k.startswith("__")})
