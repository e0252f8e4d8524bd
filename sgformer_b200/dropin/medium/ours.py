"""Drop-in replacement of the reference's medium/ours.py (medium/parse.py:2 `from ours import *`).  The GNN branch is
whatever parse.py injects (`gnn=`): a models.GCN-shaped module runs natively on the CUDA kernels, anything else is
called as given and only the attention branch, mix and fc run here."""
from sgformer_b200.medium import *  # noqa: F401,F403
from sgformer_b200.medium import SGFormer, TransConv, TransConvLayer, full_attention_conv  # noqa: F401
