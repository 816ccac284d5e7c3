"""Explicit parameter store for the synthesis path.

The reference keeps its weights implicitly in TF variable scopes and fills them with
`tf.global_variables_initializer()` followed by `Saver.restore`
(/root/reference/synthesize.py:29-41).  No checkpoint is reachable offline, so this
module provides (a) the initialiser half -- seeded draws that follow the reference's
initialisers (modules.py:35 truncated_normal(0, 0.1); modules.py:132,185,238
variance_scaling_initializer(); zero biases; LN gamma=1, beta=0) -- and (b) a plain
name -> array dictionary keyed by the TF variable names (SURVEY.md App. C) that a
checkpoint reader can fill later.

Everything here is host-side numpy; the device copy lives inside the C library
handle (see `engine.Engine.load_params`).
"""
import numpy as np

from .arch import param_shapes


def _truncated_normal(rng, shape, stddev):
    """Normal(0, stddev) with values beyond 2 stddev re-drawn (TF semantics)."""
    out = rng.standard_normal(size=shape)
    bad = np.abs(out) > 2.0
    while bad.any():
        out[bad] = rng.standard_normal(size=int(bad.sum()))
        bad = np.abs(out) > 2.0
    return (out * stddev).astype(np.float32)


def _fan_in(shape):
    # tf.contrib.layers.variance_scaling_initializer: fan_in = shape[-2] * receptive field
    rf = 1
    for s in shape[:-2]:
        rf *= s
    return float(shape[-2] * rf)


def init_params(seed=0, scheme="tf_default"):
    """Draw every variable on the path.

    scheme="tf_default": exactly the reference initialisers (bias 0, gamma 1, beta 0),
        under which the bias/gamma/beta code paths are identities.
    scheme="perturbed": same kernels, plus gamma = 1 + 0.1 n, beta = 0.1 n,
        bias = 0.1 n (n ~ N(0,1)) so those code paths are exercised (SURVEY.md 8c).
    """
    if scheme not in ("tf_default", "perturbed"):
        raise ValueError("unknown scheme %r" % (scheme,))
    params = {}
    for idx, (name, shape) in enumerate(sorted(param_shapes().items())):
        rng = np.random.default_rng([seed, idx])
        leaf = name.rsplit("/", 1)[-1]
        if leaf == "lookup_table":
            v = _truncated_normal(rng, shape, 0.1)
        elif leaf == "kernel":
            v = _truncated_normal(rng, shape, np.sqrt(1.3 * 2.0 / _fan_in(shape)))
        elif leaf == "gamma":
            v = np.ones(shape, np.float32)
            if scheme == "perturbed":
                v = v + 0.1 * rng.standard_normal(size=shape).astype(np.float32)
        else:  # bias, beta
            v = np.zeros(shape, np.float32)
            if scheme == "perturbed":
                v = 0.1 * rng.standard_normal(size=shape).astype(np.float32)
        params[name] = np.ascontiguousarray(v, dtype=np.float32)
    return params


def check_params(params):
    """Raise if `params` does not hold exactly the variables of the path."""
    want = param_shapes()
    missing = sorted(set(want) - set(params))
    extra = sorted(set(params) - set(want))
    if missing or extra:
        raise KeyError("parameter set mismatch: missing=%s extra=%s" % (missing[:4], extra[:4]))
    for k, shp in want.items():
        if tuple(params[k].shape) != tuple(shp):
            raise ValueError("%s: shape %s, expected %s" % (k, params[k].shape, shp))
    return True


def num_params(prefix=""):
    return int(sum(int(np.prod(s)) for k, s in param_shapes().items() if k.startswith(prefix)))


def synthetic_text(batch, n_chars=100, seed=0, first_index=0):
    """Synthetic fixed-length character batches (BASELINE.md section 3): ids uniform in
    [2, 31] for n_chars positions, then E (=1), then P (=0) padding to max_N.
    Row i is drawn from seed (seed, first_index + i) so shards of a global batch are
    independent of how it is split across ranks."""
    from .hyperparams import Hyperparams as hp
    L = np.zeros((batch, hp.max_N), np.int32)
    for i in range(batch):
        rng = np.random.default_rng([seed, first_index + i])
        L[i, :n_chars] = rng.integers(2, len(hp.vocab), size=n_chars)
        L[i, n_chars] = 1
    return L


def synthetic_bucket(batch, N, T, seed=0):
    """A synthetic length-bucketed batch in the shape trainer.bucketed_batches emits (dynamic padding to the longest
    member): L (batch, N) int32 and mels (batch, T, n_mels).  Row 0 is the longest member (N - 1 ids uniform in [2, 31],
    then E); row b has N - bN/(2 batch) positions and T - bT/(2 batch) frames uniform in [0, 1), zero padded after them."""
    from .hyperparams import Hyperparams as hp
    rng = np.random.default_rng([seed, N, T])
    L = np.zeros((batch, N), np.int32)
    mels = np.zeros((batch, T, hp.n_mels), np.float32)
    for b in range(batch):
        n, t = N - (b * N) // (2 * batch), T - (b * T) // (2 * batch)
        L[b, :n - 1] = rng.integers(2, len(hp.vocab), size=n - 1)
        L[b, n - 1] = 1
        mels[b, :t] = rng.uniform(0, 1, (t, hp.n_mels))
    return L, mels
