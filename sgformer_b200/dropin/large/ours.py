"""Drop-in replacement of the reference's large/ours.py: put this directory ahead of the script directory on sys.path
(python -m sgformer_b200.launch --variant large <reference>/large/main-batch.py ...) and `from ours import *`
(large/parse.py:2) resolves to the H100 implementation; main.py / main-batch.py / parse.py stay byte-unchanged."""
from sgformer_b200.large import *  # noqa: F401,F403
from sgformer_b200.large import GraphConv, GraphConvLayer, SGFormer, TransConv, TransConvLayer  # noqa: F401
