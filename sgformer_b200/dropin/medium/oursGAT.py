"""Drop-in replacement of the reference's medium/ablation/oursGAT.py (medium/ablation/parse.py, `--method ours --use_graph
--attention gat`)."""
from sgformer_b200.ablation_gat import *  # noqa: F401,F403
from sgformer_b200.ablation_gat import GATAttention, SGFormerGAT, TransConv, TransConvLayer, TransConvLayerGAT  # noqa: F401
