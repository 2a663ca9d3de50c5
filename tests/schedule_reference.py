"""CPU restatement of a parameter schedule: the oracle booster with its parameters changed between rounds, the way
Booster.set_param changes the engine's (DESIGN.md 2 item 22).  Test infrastructure only."""
import ctypes as C

import numpy as np

from oracle import oracle as O


def set_params(bst, changes):
    """Train the next rounds of oracle booster `bst` with `changes` applied to its parameters.  or_model_new copies the
    OrParams it is given into the first member of its OrModel; the new block is written there, so the trees already
    grown, the margin and the tree count that seeds the sampling stay as they are."""
    bst.params.update(changes)
    bst.p = O.make_params(bst.params)
    C.memmove(bst.h, C.byref(bst.p), C.sizeof(O.OrParams))


def train(params, X, y, num_boost_round, schedule):
    """oracle.train with schedule[r] (a dict) applied before round r.  params must carry base_score."""
    X = np.ascontiguousarray(X, np.float32)
    cuts = O.Cuts.from_data(X, int(params.get("max_bin", 256)))
    bins = cuts.bin(X)
    bst = O.Booster(params, cuts)
    bst.init_margin(X.shape[0])
    for r in range(num_boost_round):
        if r in schedule:
            set_params(bst, schedule[r])
        bst.boost(bins, y)
    return bst
