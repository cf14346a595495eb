from .activation import *  # noqa: F401,F403
from .attention import *  # noqa: F401,F403
from .conv import *  # noqa: F401,F403
from .downsample import *  # noqa: F401,F403
from .dropblock import *  # noqa: F401,F403
from .lambda_layer import *  # noqa: F401,F403
from .loss import *  # noqa: F401,F403
