# Same import surface as the reference's model_zoo/__init__.py:1-3, restricted to the backbones this
# hot path covers (the other backbones are out of scope, SURVEY.md §2.2): BNInception, and InceptionV3 at test time.
from .bninception import BNInception  # noqa: F401
from .inception_v3 import InceptionV3  # noqa: F401
