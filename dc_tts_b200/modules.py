"""Building blocks with the reference's signatures (/root/reference/modules.py), each
executed as fused sm_90a kernels through the C-ABI.

`embed` :13, `normalize` :45, `conv1d` :91, `hc` :143, `conv1d_transpose` :199 keep the
reference argument names and order.  Variables are not created here: they live in the
engine's committed parameter set and are selected by the enclosing `variable_scope`
stack plus the `scope=` argument, reproducing the TF variable names (SURVEY.md App. C).
`highwaynet` (:67) is dead code in the reference and is not provided.

Only inference semantics exist (training=False, dropout = identity: modules.py:139,195,245);
asking for training-mode dropout raises instead of silently differing.
"""
import contextlib
import threading

from .engine import get_engine

_tls = threading.local()


def _stack():
    if not hasattr(_tls, "scopes"):
        _tls.scopes = []
    return _tls.scopes


@contextlib.contextmanager
def variable_scope(name, reuse=None):
    """Stand-in for tf.variable_scope: only contributes to variable names."""
    _stack().append(name)
    try:
        yield
    finally:
        _stack().pop()


def _full(scope):
    return "/".join(_stack() + [scope])


class nn:
    """Activation tokens in place of tf.nn.relu / tf.nn.sigmoid callables."""
    relu = "relu"
    sigmoid = "sigmoid"


def _act_code(fn):
    if fn is None:
        return 0
    name = fn if isinstance(fn, str) else getattr(fn, "__name__", "")
    if name == "relu":
        return 1
    raise NotImplementedError("activation %r: the synthesis path only uses None / relu" % (fn,))


def _no_dropout(dropout_rate, training):
    if training and dropout_rate:
        raise NotImplementedError("training-mode dropout is outside the synthesis hot path (SURVEY.md 8)")


def embed(inputs, vocab_size, num_units, zero_pad=True, scope="embedding", reuse=None):
    """modules.py:13-42. ids (B,N) -> (B,N,num_units); id 0 maps to zeros."""
    if not zero_pad:
        raise NotImplementedError("embed: the path always uses zero_pad=True (modules.py:36)")
    out = get_engine().embed(_full(scope), inputs)
    if out.shape[-1] != num_units:
        raise ValueError("embed: num_units does not match the committed table")
    return out


def normalize(inputs, scope="normalize", reuse=None):
    """modules.py:45-64. Layer-norm over the last axis, eps 1e-12."""
    return get_engine().normalize(_full(scope), inputs)


def conv1d(inputs, filters=None, size=1, rate=1, padding="SAME", dropout_rate=0, use_bias=True,
           activation_fn=None, training=True, scope="conv1d", reuse=None):
    """modules.py:91-141: conv (+bias) -> LN -> activation, one fused block."""
    _no_dropout(dropout_rate, training)
    if not use_bias:
        raise NotImplementedError("conv1d: use_bias=False is never used on the path")
    if padding.lower() not in ("same", "causal"):
        raise NotImplementedError("conv1d: padding %r is never used on the path" % padding)
    if filters is None:
        filters = inputs.shape[-1]
    return get_engine().conv1d(_full(scope), inputs, filters, rate, padding.lower() == "causal",
                               _act_code(activation_fn))


def hc(inputs, filters=None, size=1, rate=1, padding="SAME", dropout_rate=0, use_bias=True,
       activation_fn=None, training=True, scope="hc", reuse=None):
    """modules.py:143-197: highway conv block, one fused block."""
    _no_dropout(dropout_rate, training)
    if activation_fn is not None:
        raise NotImplementedError("hc: every caller leaves activation_fn=None (networks.py)")
    if padding.lower() not in ("same", "causal"):
        raise NotImplementedError("hc: padding %r is never used on the path" % padding)
    return get_engine().hc(_full(scope), inputs, rate, padding.lower() == "causal")


def conv1d_transpose(inputs, filters=None, size=3, stride=2, padding='same', dropout_rate=0, use_bias=True,
                     activation=None, training=True, scope="conv1d_transpose", reuse=None):
    """modules.py:199-247: stride-2 transposed conv -> LN (time axis doubles)."""
    _no_dropout(dropout_rate, training)
    if size != 3 or stride != 2 or padding.lower() != "same" or activation is not None:
        raise NotImplementedError("conv1d_transpose: only size=3, stride=2, 'same', no activation (networks.py:242)")
    return get_engine().conv1d_transpose(_full(scope), inputs)
