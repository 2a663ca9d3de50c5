"""DART (booster="dart") on top of the oracle: the drop draw, the weight normalisation and the weighted margins in
NumPy, the trees grown by the oracle (`train`) from gradients taken at the drop margin.

What the engine implements (csrc/round.cu dart_drop_set / dart_prepare, csrc/dart_kernel.cu; DESIGN.md 2), written out
independently so that the GPU tests can replay a trained model round by round:
  * draw u_j = hash4(seed, r, j, SCOPE_DART) / 2^32 (the counter-based hash of csrc/sampling.cuh), r = rounds already
    in the model; j = 0xFFFFFFFF decides skip_drop, j = 0xFFFFFFFE the one_drop pick;
  * a row's margin is base + sum over trees in order of fl(w_t * leaf_t), each add a float32 multiply then add;
  * the drop margin leaves the round's dropped trees out, the full margin keeps every tree.
Tree traversal is on the bin matrix (bin <= split_bin -> left, missing bin 255 of a feature with missing values ->
default direction, categorical code in the node's set -> right), the walk the engine's margin rebuild does.
`train` grows a model round by round with the oracle's own tree growth: the drop set of the round, the drop margin from
the oracle's trees so far, the gradients at it (the oracle's for its objectives, tests/objective_reference.py's for the
others) handed to oracle.Booster.boost as custom gradients, then the normalisation.  The weights are kept here."""
import numpy as np

F32 = np.float32
_DRAW_KEYS = ("rate_drop", "skip_drop", "sample_type", "one_drop")

SCOPE_DART = 2
_M64 = (1 << 64) - 1


def _mix64(x):
    x &= _M64
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & _M64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & _M64
    x ^= x >> 31
    return x


def hash4(seed, a, b, c):
    h = _mix64(((seed & 0xFFFFFFFF) * 0x9E3779B97F4A7C15 + (a & 0xFFFFFFFF)) & _M64)
    h = _mix64((h + (b & 0xFFFFFFFF)) & _M64)
    h = _mix64((h + (c & 0xFFFFFFFF)) & _M64)
    return h >> 32


def draw(seed, r, j):
    return hash4(seed, r, j, SCOPE_DART) * 2.0 ** -32


def drop_set(weights, r, seed=0, rate_drop=0.0, skip_drop=0.0, sample_type="uniform", one_drop=0):
    """Indices of the trees round r drops, given the weights of the T trees before it."""
    w = np.asarray(weights, np.float32)
    T = w.size
    if T == 0:
        return []
    if skip_drop > 0 and draw(seed, r, 0xFFFFFFFF) < skip_drop:
        return []
    S = np.float32(0.0)
    for x in w:                                  # binary32, in tree order
        S = np.float32(S + x)
    out = []
    for t in range(T):
        thr = rate_drop * T * float(w[t]) / float(S) if sample_type == "weighted" else rate_drop
        if draw(seed, r, t) < thr:
            out.append(t)
    if one_drop and not out:
        v = draw(seed, r, 0xFFFFFFFE)
        if sample_type == "weighted":
            cum, pick = 0.0, T - 1
            for t in range(T):
                cum += float(w[t])
                if cum > v * float(S):
                    pick = t
                    break
        else:
            pick = min(T - 1, int(np.floor(v * T)))
        out = [pick]
    return out


def normalize(weights, dropped, eta, n_new, normalize_type="tree"):
    """Weights after a round that dropped `dropped` and grew n_new trees (Dart::NormalizeTrees as DESIGN.md 2 states)."""
    w = np.array(weights, np.float32)
    lr = float(np.float32(float(np.float32(eta)) / n_new))
    k = len(dropped)
    if k == 0:
        return np.concatenate([w, np.ones(n_new, np.float32)])
    if normalize_type == "forest":
        f = np.float32(1.0 / (1.0 + lr))
        new = f
    else:
        f = np.float32(k / (k + lr))
        new = np.float32(1.0 / (k + lr))
    for t in dropped:
        w[t] = np.float32(w[t] * f)
    return np.concatenate([w, np.full(n_new, new, np.float32)])


def replay_weights(n_rounds, eta, n_new, r0=0, weights=(), **kw):
    """Weights and drop sets of rounds r0 .. r0 + n_rounds - 1, starting from `weights` (the model before r0)."""
    w = np.asarray(weights, np.float32)
    drops = []
    for r in range(r0, r0 + n_rounds):
        d = drop_set(w, r, **{k: v for k, v in kw.items() if k != "normalize_type"})
        drops.append(d)
        w = normalize(w, d, eta, n_new, kw.get("normalize_type", "tree"))
    return w, drops


def _as_dict(tree):
    if isinstance(tree, dict):
        return tree
    return {k: getattr(tree, k) for k in ("left", "right", "split_feature", "split_bin", "default_left", "value",
                                          "split_type", "cat_bits")}


def leaves_on_bins(tree, bins, has_missing):
    """Leaf node id of every row of the bin matrix `bins` ([n][F] uint8)."""
    tree = _as_dict(tree)
    n = bins.shape[0]
    nid = np.zeros(n, np.int64)
    st = tree.get("split_type")
    while True:
        f = tree["split_feature"][nid]
        inner = f >= 0
        if not inner.any():
            return nid
        rows = np.nonzero(inner)[0]
        nd, ff = nid[rows], f[rows]
        b = bins[rows, ff].astype(np.int64)
        left = b <= tree["split_bin"][nd]
        if st is not None:
            cat = st[nd] != 0
            if cat.any():
                words = tree["cat_bits"][nd[cat], b[cat] >> 5]
                left[cat] = ((words >> (b[cat] & 31).astype(np.uint32)) & 1) == 0
        miss = (b == 255) & (np.asarray(has_missing)[ff] != 0)
        left[miss] = tree["default_left"][nd[miss]] != 0
        nid[rows] = np.where(left, tree["left"][nd], tree["right"][nd])


def margins(trees, weights, bins, has_missing, base, K=1, npt=1, skip=()):
    """base ([n][K] float32) + the ordered weighted leaf sums, leaving out the trees in `skip`."""
    m = np.array(base, np.float32).reshape(bins.shape[0], K).copy()
    skip = set(skip)
    for t, tree in enumerate(trees):
        if t in skip:
            continue
        v = _as_dict(tree)["value"][leaves_on_bins(tree, bins, has_missing)].astype(np.float32)
        c = (t // npt) % K
        m[:, c] = m[:, c] + np.float32(weights[t]) * v
    return m


class Model:
    """A DART model grown by `train`: tree(i) in the engine's order (the parallel trees of a class next to each other),
    the weights, and the train matrix's bins."""

    def __init__(self, bst, K, npt, weights, drops, bins, has_missing, base):
        self.bst, self.K, self.npt = bst, K, npt
        self.weights, self.drops, self.bins, self.has_missing, self.base = weights, drops, bins, has_missing, base
        self._trees = []

    @property
    def num_trees(self):
        return self.bst.num_trees

    def tree(self, i):
        while len(self._trees) <= i:   # finished trees never change: fetch each once
            j = len(self._trees)
            r, rem = divmod(j, self.K * self.npt)
            k, p = divmod(rem, self.npt)
            self._trees.append(self.bst.tree(r * self.K * self.npt + p * self.K + k))   # the oracle grows class-major
        return self._trees[i]

    def trees(self):
        return [self.tree(i) for i in range(self.num_trees)]

    def margin(self, skip=()):
        return margins(self.trees(), self.weights, self.bins, self.has_missing, self.base, self.K, self.npt, skip)


def train(oracle, params, X, y, rounds, weight=None, is_cat=None, base_margin=None):
    """`rounds` DART rounds grown by the oracle.  params: the engine's (booster=dart, the DART keys, an explicit
    base_score); num_parallel_tree > 1 grows npt oracle rounds per round from the same gradients with eta / npt."""
    from tests import objective_reference as O
    obj = params.get("objective", "reg:squarederror")
    K = int(params.get("num_class", 1)) if obj.startswith("multi:") else 1
    npt = int(params.get("num_parallel_tree", 1))
    eta = float(params.get("eta", 0.3))
    X = np.ascontiguousarray(X, F32)
    y = np.ascontiguousarray(y, F32)
    op = {k: v for k, v in params.items() if k not in _DRAW_KEYS + ("normalize_type", "booster", "num_parallel_tree")}
    if npt > 1:
        op["eta"] = float(F32(eta) / F32(npt))
    own = obj in oracle.OBJECTIVES
    if not own:   # an objective the oracle does not have: squared-error growth fed with the restated gradients
        b = float(F32(params["base_score"]))
        op.update(objective="reg:squarederror", base_score=O.base_margin(obj, b), max_delta_step=O.max_delta_step(params))
    cuts = oracle.Cuts.from_data(X, int(params.get("max_bin", 256)), np.nan, is_cat=is_cat, weight=weight)
    bins = cuts.bin(X)
    bst = oracle.Booster(op, cuts)
    base = bst.init_margin(X.shape[0], base_margin).copy()
    model = Model(bst, K, npt, np.zeros(0, F32), [], bins, cuts.has_missing, base)
    draw_kw = {k: params[k] for k in _DRAW_KEYS if k in params}
    for r in range(rounds):
        drop = drop_set(model.weights, r, seed=int(params.get("seed", 0)), **draw_kw)
        m = model.margin(skip=drop)
        if own:
            g, h = oracle.gradients(obj, m, y, weight, num_class=K)
        else:
            g, h, bad = O.gradients(params, m[:, 0], y, weight)
            assert not bad, "a gradient is not finite"
        for _ in range(npt):
            bst.boost(bins, y, weight, custom_g=g, custom_h=h)
        model.weights = normalize(model.weights, drop, eta, K * npt, params.get("normalize_type", "tree"))
        model.drops.append(drop)
    return model
