"""``models.vgg_128`` of the reference, served by the sm_90a implementation."""
from p2pvg_b200.models.vgg_128 import *  # noqa: F401,F403
from p2pvg_b200.models import vgg_128 as _impl

globals().update({k: v for k, v in vars(_impl).items() if not k.startswith("__")})
