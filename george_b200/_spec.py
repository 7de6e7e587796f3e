# -*- coding: utf-8 -*-
"""
Flatten a kernel-spec object tree into the POD postfix program of ``include/bgp.h``.

This is the host-side replacement for ``parse_kernel_spec`` (reference
``src/george/include/george/parser.h:14-509``): it reads exactly the attributes the reference's parser reads
(``is_kernel``, ``operator_type``, ``k1``/``k2``, ``kernel_type``, ``metric.{metric_type,ndim,axes,
get_parameter_vector(True)}``, ``blocked``/``min_block``/``max_block``, ``ndim``/``axes`` and the per-kernel
parameter attributes) and raises the same exception types (``ValueError`` for an invalid kernel or an
unknown id, ``RuntimeError`` for a dimension mismatch between the operands of ``+``/``*``).
"""

import ctypes as C

import numpy as np

BGP_MAX_DIM = 8
BGP_MAX_METRIC = 36
BGP_MAX_NODES = 32

OP_KERNEL, OP_SUM, OP_PRODUCT = 0, 1, 2


class KernelNode(C.Structure):
    _fields_ = [
        ("op", C.c_int32), ("kernel_type", C.c_int32), ("metric_type", C.c_int32), ("ndim", C.c_int32),
        ("naxes", C.c_int32), ("blocked", C.c_int32), ("n_params", C.c_int32), ("n_metric", C.c_int32),
        ("axes", C.c_int32 * BGP_MAX_DIM),
        ("params", C.c_double * 4),
        ("metric", C.c_double * BGP_MAX_METRIC),
        ("min_block", C.c_double * BGP_MAX_DIM),
        ("max_block", C.c_double * BGP_MAX_DIM),
    ]


class KernelSpec(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("ndim", C.c_int32), ("nodes", KernelNode * BGP_MAX_NODES)]


class HodlrOpts(C.Structure):
    _fields_ = [
        ("min_size", C.c_int32), ("seed", C.c_int32), ("tol", C.c_double), ("rng_mode", C.c_int32),
        ("rank_capacity", C.c_int32), ("shard_rank", C.c_int32), ("shard_count", C.c_int32), ("exhaust_mode", C.c_int32),
    ]


class HodlrNodeInfo(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("start", "size", "half", "is_leaf", "parent", "direction", "depth", "rank",
                                          "rng_draws", "dense_fallback")]


# kernel_type -> (stationary, ordered attribute names handed to the C++ constructor in parser.h, #hyper-parameters)
#   parser.h:42-60 Linear, 62-124 RationalQuadratic, 126-185 Exp, 187-205 LocalGaussian, 207-223 Empty,
#   225-242 Cosine, 244-303 Matern52, 305-323 ExpSine2, 325-342 Constant, 344-403 ExpSquared,
#   405-464 Matern32, 466-484 Polynomial, 486-503 DotProduct
_KERNELS = {
    0: (False, ("log_gamma2", "order"), 1),
    1: (True, ("log_alpha",), 1),
    2: (True, (), 0),
    3: (False, ("location", "log_width"), 2),
    4: (False, (), 0),
    5: (False, ("log_period",), 1),
    6: (True, (), 0),
    7: (False, ("gamma", "log_period"), 2),
    8: (False, ("log_constant",), 1),
    9: (True, (), 0),
    10: (True, (), 0),
    11: (False, ("log_sigma2", "order"), 1),
    12: (False, (), 0),
}


# user kernels compiled in from kernels/*.yml (tools/generate_kernels.py): parameters first, then constants, as above
try:
    from .user_kernels import USER_KERNEL_TABLE as _USER
except ImportError:  # pragma: no cover
    _USER = []
for _name, _kt, _stat, _params, _consts, _doc in _USER:
    _KERNELS[_kt] = (_stat, tuple(_params) + tuple(_consts), len(_params))


class DimensionMismatch(RuntimeError):
    """What pybind11 turns ``george::dimension_mismatch`` (exceptions.h:8-12) into."""


def _emit(obj, nodes):
    if not hasattr(obj, "is_kernel"):
        raise ValueError("invalid kernel")
    if not bool(obj.is_kernel):
        nd1 = _emit(obj.k1, nodes)
        nd2 = _emit(obj.k2, nodes)
        if nd1 != nd2:
            raise DimensionMismatch("dimension mismatch")
        op = int(obj.operator_type)
        if op not in (0, 1):
            raise ValueError("unrecognized operator")
        node = KernelNode()
        node.op = OP_SUM if op == 0 else OP_PRODUCT
        node.kernel_type = -1
        node.metric_type = -1
        node.ndim = nd1
        nodes.append(node)
        return nd1

    ktype = int(obj.kernel_type)
    if ktype not in _KERNELS:
        raise ValueError("unrecognized kernel")
    stationary, attrs, n_params = _KERNELS[ktype]
    node = KernelNode()
    node.op = OP_KERNEL
    node.kernel_type = ktype
    node.n_params = n_params
    for i, a in enumerate(attrs):
        node.params[i] = float(getattr(obj, a))
    if stationary:
        metric = obj.metric
        node.metric_type = int(metric.metric_type)
        if node.metric_type not in (0, 1, 2):
            raise ValueError("unrecognized metric")
        ndim = int(metric.ndim)
        axes = [int(a) for a in list(metric.axes)]
        vec = np.asarray(metric.get_parameter_vector(True), dtype=np.float64)
        if len(vec) > BGP_MAX_METRIC:
            raise ValueError("metric has too many parameters for the device program")
        node.n_metric = len(vec)
        for i, v in enumerate(vec):
            node.metric[i] = float(v)
        node.blocked = 1 if bool(obj.blocked) else 0
        mn = np.asarray(obj.min_block, dtype=np.float64)
        mx = np.asarray(obj.max_block, dtype=np.float64)
    else:
        node.metric_type = -1
        node.n_metric = 0
        ndim = int(obj.ndim)
        axes = [int(a) for a in list(obj.axes)]
        mn = mx = None
    if len(axes) > BGP_MAX_DIM:
        raise ValueError("kernels acting on more than {0} axes are not supported on the device".format(BGP_MAX_DIM))
    node.ndim = ndim
    node.naxes = len(axes)
    for i, a in enumerate(axes):
        node.axes[i] = a
        if mn is not None:
            node.min_block[i] = float(mn[i])
            node.max_block[i] = float(mx[i])
    nodes.append(node)
    return ndim


def flatten(kernel_spec):
    """Return a ``KernelSpec`` ctypes struct for the given kernel object."""
    nodes = []
    ndim = _emit(kernel_spec, nodes)
    if len(nodes) > BGP_MAX_NODES:
        raise ValueError("kernel expression has more than {0} nodes".format(BGP_MAX_NODES))
    spec = KernelSpec()
    spec.n_nodes = len(nodes)
    spec.ndim = ndim
    for i, n in enumerate(nodes):
        spec.nodes[i] = n
    return spec


def num_params(spec):
    return sum(spec.nodes[i].n_params + spec.nodes[i].n_metric for i in range(spec.n_nodes))


def parameter_slots(spec):
    """``(node, field, index)`` of every parameter slot of ``spec``, in the order :func:`patch_specs` fills them: node
    by node, a leaf's ``params[:n_params]`` followed by its ``metric[:n_metric]``."""
    slots = []
    for i in range(spec.n_nodes):
        node = spec.nodes[i]
        if node.op != OP_KERNEL:
            continue
        slots.extend((i, "params", j) for j in range(node.n_params))
        slots.extend((i, "metric", j) for j in range(node.n_metric))
    return slots


def patch_specs(template, params):
    """``B`` copies of ``template`` (a :func:`flatten` result) with their parameter slots overwritten by the rows of
    ``params`` (``(B, num_params(template))``); returns a contiguous ``KernelSpec * B`` array.

    It relies on the slot order matching the kernel's full parameter vector: for every kernel ``k``,
    ``k.get_parameter_vector(include_frozen=True)`` is the concatenation over the leaves of ``flatten(k)``, in node
    order, of ``params[:n_params]`` and ``metric[:n_metric]``.  So row ``b`` patched in gives, byte for byte,
    ``flatten(k)`` after ``k.set_parameter_vector(params[b], include_frozen=True)``: everything else in the program
    (structure, axes, blocks, constants such as a polynomial's order) does not depend on the parameter values.
    ``bgp_dense_batch_log_likelihood`` patches the same slots in the same order."""
    params = np.asarray(params, dtype=np.float64)
    slots = parameter_slots(template)
    if params.ndim != 2 or params.shape[1] != len(slots):
        raise ValueError("params must have shape (B, {0})".format(len(slots)))
    out = (KernelSpec * params.shape[0])()
    for b in range(params.shape[0]):
        C.memmove(C.byref(out[b]), C.byref(template), C.sizeof(KernelSpec))
        row = params[b]
        for k, (i, field, j) in enumerate(slots):
            getattr(out[b].nodes[i], field)[j] = float(row[k])
    return out
