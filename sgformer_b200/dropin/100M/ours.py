"""Drop-in replacement of the reference's 100M/ours.py (100M/parse.py:1 `from ours import *`)."""
from sgformer_b200.hundred_m import *  # noqa: F401,F403
from sgformer_b200.hundred_m import (GraphConv, GraphConvLayer, SGFormer, TransConv, TransConvLayer,  # noqa: F401
                                     full_attention_conv)
