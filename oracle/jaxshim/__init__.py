"""A minimal numpy-backed stand-in for the parts of jax / flax.linen that the reference's *loss, RoPE,
param-group, layer, ViT, DINOHead and SSLMetaArch* modules touch — TEST INFRASTRUCTURE, used only by tests/golden/make_golden.py in the build container
(where a reference checkout exists and the real jax/flax cannot be installed) to execute those reference files UNMODIFIED
and record golden vectors.  It is not a JAX implementation: only single-device, eager, float64 numpy semantics.
Third-party semantics restated here (SURVEY.md Appendix F): nn.softmax / nn.log_softmax are the max-subtracted
forms; jax.lax.psum / pmean over one device are the identity; jax.lax.cond picks a branch eagerly.
"""
from __future__ import annotations

import sys
import types

import numpy as np


class _At:
    def __init__(self, arr):
        self.arr = arr

    def __getitem__(self, idx):
        arr = self.arr

        class _Setter:
            def set(self, v):
                out = np.array(arr, copy=True).view(Arr)
                out[idx] = v
                return out
        return _Setter()


class Arr(np.ndarray):
    @property
    def at(self):
        return _At(self)

    def astype(self, dtype, *a, **k):
        if dtype is None:
            return self
        return np.ndarray.astype(self, dtype, *a, **k).view(Arr)


def _wrap(x):
    if isinstance(x, np.ndarray) and not isinstance(x, Arr):
        return x.view(Arr)
    if isinstance(x, (tuple, list)):
        return type(x)(_wrap(v) for v in x)
    return x


class _NumpyProxy(types.ModuleType):
    """jax.numpy: forwards to numpy, wraps results so `.at[...]` works."""

    def __init__(self, name, target):
        super().__init__(name)
        self._t = target

    def __getattr__(self, name):
        attr = getattr(self._t, name)
        if callable(attr) and not isinstance(attr, type):
            def f(*a, **k):
                if "dtype" in k and k["dtype"] is None:
                    k.pop("dtype")
                return _wrap(attr(*a, **k))
            return f
        if isinstance(attr, types.ModuleType):
            return _NumpyProxy(self.__name__ + "." + name, attr)
        return attr


def _fill_diagonal(a, val, inplace=True):
    out = np.array(a, copy=True)
    np.fill_diagonal(out, val)
    return out.view(Arr)


def _softmax(x, axis=-1):
    x = np.asarray(x)
    e = np.exp(x - x.max(axis=axis, keepdims=True))
    return (e / e.sum(axis=axis, keepdims=True)).view(Arr)


def _log_softmax(x, axis=-1):
    x = np.asarray(x)
    s = x - x.max(axis=axis, keepdims=True)
    return (s - np.log(np.exp(s).sum(axis=axis, keepdims=True))).view(Arr)


def _gelu(x, approximate=True):
    x = np.asarray(x)
    assert approximate
    return (0.5 * x * (1 + np.tanh(np.sqrt(2 / np.pi) * (x + 0.044715 * x ** 3)))).view(Arr)


class _Variable:
    def __init__(self, value):
        self.value = value


# --------------------------------------------------------------------------------------------------------------------
# mini flax.linen: just enough of the Module system to execute the reference's layers / ViT / DINOHead unmodified with
# externally supplied parameters.  PARAMS maps "path/to/leaf" -> array, paths follow flax naming: attribute name for
# submodules created in setup(), "<attr>_<i>" for list attributes, "<Class>_<n>" for submodules created inside an
# @nn.compact __call__, "layers_<i>" for nn.Sequential (SURVEY.md Appendix C / F).
PARAMS: dict = {}
_STACK: list = []


def _adopt(parent, child, name):
    if isinstance(child, Module) and child.__dict__.get("_parent") is None and child is not parent:
        object.__setattr__(child, "_parent", parent)
        object.__setattr__(child, "_name", name)


class Module:
    def __init_subclass__(cls, **kw):
        super().__init_subclass__(**kw)
        if "__call__" in cls.__dict__:
            inner = cls.__dict__["__call__"]

            def wrapped(self, *a, __inner=inner, **k):
                self._ensure_setup()
                object.__setattr__(self, "_auto", {})
                _STACK.append(self)
                try:
                    return __inner(self, *a, **k)
                finally:
                    _STACK.pop()
            cls.__call__ = wrapped

    def __init__(self, *args, **kwargs):
        d = self.__dict__
        d.update(_parent=None, _name=None, _setup_done=False, _in_setup=False, _auto={})
        fields = []
        for klass in reversed(type(self).__mro__):
            fields += [n for n in getattr(klass, "__annotations__", {}) if n not in fields]
        values = dict(zip(fields, args))
        values.update(kwargs)
        for n in fields:
            if n in values:
                setattr(self, n, values[n])
            else:
                if not hasattr(type(self), n):
                    raise TypeError(f"{type(self).__name__}: missing field {n}")
                object.__setattr__(self, n, getattr(type(self), n))   # instance attribute: plain functions stay unbound
        if _STACK and not _STACK[-1].__dict__.get("_in_setup"):          # created inside a compact __call__
            parent = _STACK[-1]
            cname = type(self).__name__
            idx = parent._auto.get(cname, 0)
            parent._auto[cname] = idx + 1
            _adopt(parent, self, f"{cname}_{idx}")

    def __setattr__(self, k, v):
        if not k.startswith("_"):
            if isinstance(v, Module):
                _adopt(self, v, k)
            elif isinstance(v, (list, tuple)):
                for i, e in enumerate(v):
                    _adopt(self, e, f"{k}_{i}")
        object.__setattr__(self, k, v)

    def __getattr__(self, k):          # only reached when normal lookup fails: attributes defined by setup()
        d = self.__dict__
        if k.startswith("__") or d.get("_setup_done") or d.get("_in_setup"):
            raise AttributeError(k)
        self._ensure_setup()
        return object.__getattribute__(self, k)

    def _ensure_setup(self):
        d = self.__dict__
        if not d["_setup_done"]:
            d["_setup_done"] = True
            if hasattr(type(self), "setup"):
                d["_in_setup"] = True
                _STACK.append(self)
                try:
                    self.setup()
                finally:
                    _STACK.pop()
                    d["_in_setup"] = False

    def _path(self):
        node, parts = self, []
        while node is not None and node.__dict__.get("_name") is not None:
            parts.append(node._name)
            node = node._parent
        return list(reversed(parts))

    def param(self, name, init_fn=None, *shape_args):
        key = "/".join(self._path() + [name])
        if key not in PARAMS:
            raise KeyError(f"parameter {key!r} not supplied")
        v = np.asarray(PARAMS[key], dtype=np.float64)
        if shape_args and isinstance(shape_args[0], (tuple, list)) and tuple(shape_args[0]) != v.shape:
            raise ValueError(f"{key}: shape {v.shape} != requested {tuple(shape_args[0])}")
        return v.view(Arr)

    def variable(self, collection, name, init_fn, *a):
        return _Variable(_wrap(init_fn(*a)))

    def make_rng(self, name):
        raise RuntimeError("rng requested on the deterministic path")


class Dense(Module):
    features: int
    use_bias: bool = True
    kernel_init: object = None
    bias_init: object = None
    dtype: object = None
    param_dtype: object = None

    def __call__(self, x):
        y = np.asarray(x) @ self.param("kernel", None, (np.shape(x)[-1], self.features))
        if self.use_bias:
            y = y + self.param("bias", None, (self.features,))
        return _wrap(np.asarray(y))


class LayerNorm(Module):
    epsilon: float = 1e-6
    use_bias: bool = True
    use_scale: bool = True
    dtype: object = None

    def __call__(self, x):
        x = np.asarray(x)
        mean = x.mean(-1, keepdims=True)
        var = np.maximum((x * x).mean(-1, keepdims=True) - mean * mean, 0.0)    # use_fast_variance
        y = (x - mean) / np.sqrt(var + self.epsilon)
        if self.use_scale:
            y = y * self.param("scale", None, (x.shape[-1],))
        if self.use_bias:
            y = y + self.param("bias", None, (x.shape[-1],))
        return _wrap(y)


class Conv(Module):
    features: int
    kernel_size: object = None
    strides: object = 1
    padding: object = "SAME"
    use_bias: bool = True

    def __call__(self, x):
        x = np.asarray(x)
        kh, kw = self.kernel_size
        assert tuple(self.strides) == (kh, kw), "shim Conv supports stride == kernel (patch embedding) only"
        b, H, W, c = x.shape
        assert H % kh == 0 and W % kw == 0
        k = self.param("kernel", None, (kh, kw, c, self.features))
        p = x.reshape(b, H // kh, kh, W // kw, kw, c).transpose(0, 1, 3, 2, 4, 5).reshape(b, H // kh, W // kw, kh * kw * c)
        y = p @ np.asarray(k).reshape(kh * kw * c, self.features)
        if self.use_bias:
            y = y + self.param("bias", None, (self.features,))
        return _wrap(y)


class Dropout(Module):
    rate: float = 0.0

    def __call__(self, x, deterministic=True):
        assert deterministic or self.rate == 0.0
        return x


class Sequential(Module):
    layers: object = None

    def __call__(self, x):
        for l in self.layers:
            x = l(x)
        return x


def _dot_product_attention(q, k, v, deterministic=True, **unused):
    """flax.linen.dot_product_attention for [batch, len, heads, dim]: softmax((q / sqrt(dim)) k^T) v, no mask/dropout."""
    q, k, v = np.asarray(q), np.asarray(k), np.asarray(v)
    s = np.einsum("bqhd,bkhd->bhqk", q / np.sqrt(q.shape[-1]), k)
    s = s - s.max(-1, keepdims=True)
    a = np.exp(s)
    a = a / a.sum(-1, keepdims=True)
    return _wrap(np.einsum("bhqk,bkhd->bqhd", a, v))


def _initializer(*a, **k):
    return lambda *aa, **kk: None


def install():
    """Put the stand-ins into sys.modules as `jax`, `jax.numpy`, `jax.lax`, `flax`, `flax.linen`, ..."""
    jnp = _NumpyProxy("jax.numpy", np)
    jnp.fill_diagonal = _fill_diagonal
    jnp.ndarray = np.ndarray
    jnp.float32, jnp.float16, jnp.bfloat16 = np.float32, np.float16, np.float32
    jnp.inf, jnp.nan, jnp.dtype = np.inf, np.nan, np.dtype

    jax = types.ModuleType("jax")
    jax.numpy = jnp
    jax.device_count = lambda: 1
    jax.local_device_count = lambda: 1
    lax = types.ModuleType("jax.lax")
    lax.psum = lambda x, axis_name=None: x
    lax.pmean = lambda x, axis_name=None: x
    lax.cond = lambda pred, t, f, operand=None: (t if pred else f)(operand)
    lax.axis_index = lambda name: 0

    def dynamic_slice_in_dim(operand, start_index, slice_size, axis=0):
        idx = [slice(None)] * np.ndim(operand)
        idx[axis] = slice(int(start_index), int(start_index) + int(slice_size))
        return _wrap(np.asarray(operand)[tuple(idx)])
    lax.dynamic_slice_in_dim = dynamic_slice_in_dim
    jax.lax = lax
    jnn = types.ModuleType("jax.nn")
    jinit = types.ModuleType("jax.nn.initializers")
    jinit.truncated_normal = _initializer
    jnn.initializers = jinit
    jnn.gelu = _gelu
    jax.nn = jnn
    jrandom = types.ModuleType("jax.random")
    jax.random = jrandom
    jtu = types.ModuleType("jax.tree_util")

    def tree_map(fn, tree, *rest, is_leaf=None):
        if isinstance(tree, dict):
            return {k: tree_map(fn, v, *[r[k] for r in rest], is_leaf=is_leaf) for k, v in tree.items()}
        return fn(tree, *rest)
    jtu.tree_map = tree_map

    def tree_leaves(tree):
        if isinstance(tree, dict):
            return [l for v in tree.values() for l in tree_leaves(v)]
        return [tree]
    jtu.tree_leaves = tree_leaves
    jax.tree_util = jtu
    jax.vmap = lambda f: (lambda x: np.stack([f(r) for r in x]))

    flax = types.ModuleType("flax")
    nn = types.ModuleType("flax.linen")
    nn.Module = Module
    nn.softmax, nn.log_softmax, nn.gelu = _softmax, _log_softmax, _gelu
    nn.compact = lambda f: f
    inits = types.ModuleType("flax.linen.initializers")
    for n in ("lecun_normal", "normal", "constant", "truncated_normal"):
        setattr(inits, n, _initializer)
    inits.ones = _initializer()
    inits.zeros = _initializer()
    nn.initializers = inits
    nn.Dense, nn.LayerNorm, nn.Conv, nn.Dropout, nn.Sequential = Dense, LayerNorm, Conv, Dropout, Sequential
    nn.dot_product_attention = _dot_product_attention
    for n in ("BatchNorm", "make_causal_mask"):
        setattr(nn, n, type(n, (), {}))
    nn.silu = lambda x: _wrap(np.asarray(x) / (1.0 + np.exp(-np.asarray(x))))        # jax.nn.silu = x * sigmoid(x)

    class Partitioned:                     # flax.linen.Partitioned: a boxed value plus its per-axis mesh names
        def __init__(self, value=None, names=None, mesh=None):
            self.value, self.names, self.mesh = value, names, mesh
    nn.Partitioned = Partitioned
    # one device: gather/shard of un-partitioned leaves is the identity, so the FSDP wrapper returns its target
    nn.map_variables = lambda target, *a, **k: target
    flax.linen = nn
    tu = types.ModuleType("flax.traverse_util")

    def flatten_dict(d, sep=None, _pre=()):
        out = {}
        for k, v in d.items():
            if isinstance(v, dict):
                out.update(flatten_dict(v, None, _pre + (k,)))
            else:
                out[_pre + (k,)] = v
        if sep is not None and not _pre:
            out = {sep.join(k): v for k, v in out.items()}
        return out

    def unflatten_dict(d, sep=None):
        out = {}
        for k, v in d.items():
            parts = k.split(sep) if sep is not None else list(k)
            cur = out
            for p in parts[:-1]:
                cur = cur.setdefault(p, {})
            cur[parts[-1]] = v
        return out
    tu.flatten_dict, tu.unflatten_dict = flatten_dict, unflatten_dict
    flax.traverse_util = tu
    dlpack = types.ModuleType("jax.dlpack")

    def from_dlpack(capsule):
        import torch
        t = torch.utils.dlpack.from_dlpack(capsule)
        return _wrap((t.float() if t.dtype == torch.bfloat16 else t).numpy())
    dlpack.from_dlpack = from_dlpack
    jax.dlpack = dlpack
    sys.modules["jax.dlpack"] = dlpack
    sharding = types.ModuleType("jax.sharding")
    for n in ("NamedSharding", "PartitionSpec", "Mesh"):
        setattr(sharding, n, type(n, (), {"__init__": lambda self, *a, **k: None}))
    jax.sharding = sharding
    jax.__path__ = []           # lets `import jax.<sub>` resolve through sys.modules
    mods = {"jax.sharding": sharding}
    sys.modules.update(mods)
    mods = {"jax.sharding": sharding, "jax": jax, "jax.numpy": jnp, "jax.lax": lax, "jax.nn": jnn, "jax.nn.initializers": jinit,
            "jax.random": jrandom, "jax.tree_util": jtu, "flax": flax, "flax.linen": nn,
            "flax.linen.initializers": inits, "flax.traverse_util": tu}
    sys.modules.update(mods)
    return mods
