"""GPU mirrors of ``filterpy.discrete_bayes``: the drop-ins ``normalize`` / ``update`` / ``predict`` and their bank
forms over ``pdf[B, M]``, one histogram filter per row."""
from .discrete_bayes import (normalize, update, predict, normalize_bank, update_bank, predict_bank,  # noqa: F401
                             predict_update_bank)
