"""models.dcgan_64 of the reference, served by the sm_90a implementation."""
from p2pvg_b200.models.dcgan_64 import *  # noqa: F401,F403
from p2pvg_b200.models import dcgan_64 as _impl

globals().update({k: v for k, v in vars(_impl).items() if not k.startswith("__")})
