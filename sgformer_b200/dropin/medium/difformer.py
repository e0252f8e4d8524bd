"""Drop-in replacement of the reference's medium/difformer.py (medium/parse.py:4 `from difformer import *`)."""
from sgformer_b200.difformer import *  # noqa: F401,F403
