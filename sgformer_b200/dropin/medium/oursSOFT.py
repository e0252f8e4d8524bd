"""Drop-in replacement of the reference's medium/ablation/oursSOFT.py (medium/ablation/parse.py, `--method ours --attention
softmax`)."""
from sgformer_b200.ablation import *  # noqa: F401,F403
from sgformer_b200.ablation import SGFormerSOFT, TransConv, TransConvLayer, softmax_attention  # noqa: F401
