from wsl4mis_b200.networks.discriminator import *  # noqa: F401,F403
from wsl4mis_b200.networks.discriminator import FCDiscriminator  # noqa: F401
