# -*- coding: utf-8 -*-
"""GP.grad_predict on the host: the argument checks that run before any device call, the mean-model restriction, the
shape checks of KernelInterface.x1_gradient_matvec, and the error raised without a device."""
import numpy as np
import pytest


def _gp(kernel, n=5, **kw):
    import george_b200 as george
    gp = george.GP(kernel, **kw)
    gp._x = np.linspace(0, 1, n)[:, None] if kernel.ndim == 1 else np.zeros((n, kernel.ndim))
    gp._yerr2 = np.zeros(n)  # what compute() would leave, without touching the device
    return gp


def test_not_computed_raises():
    import george_b200 as george
    from george_b200 import kernels
    gp = george.GP(1.0 * kernels.ExpSquaredKernel(1.0))
    for kw in (dict(), dict(return_var=True)):
        with pytest.raises(RuntimeError, match="You need to compute the model first"):
            gp.grad_predict(np.zeros(3), np.zeros(4), **kw)


def test_non_constant_mean_raises_before_device_work():
    from george_b200 import kernels
    from george_b200.modeling import Model

    class Line(Model):
        parameter_names = ("m", "b")

        def get_value(self, x):
            return self.m * x + self.b

    gp = _gp(1.0 * kernels.ExpSquaredKernel(1.0), mean=Line(m=1.0, b=0.0))
    with pytest.raises(NotImplementedError, match="constant mean"):
        gp.grad_predict(np.zeros(5), np.zeros(4))
    import george_b200 as george
    with pytest.raises(NotImplementedError):  # not computed either: the mean is checked first
        george.GP(1.0 * kernels.ExpSquaredKernel(1.0), mean=Line(m=1.0, b=0.0)).grad_predict(np.zeros(3), np.zeros(2))


def test_dimension_checks_run_before_device_work():
    from george_b200 import kernels
    gp = _gp(1.0 * kernels.ExpSquaredKernel(1.0))
    with pytest.raises(ValueError, match="Dimension mismatch"):
        gp.grad_predict(np.zeros(5), np.zeros((4, 2)))
    gp = _gp(kernels.ExpSquaredKernel(1.0, ndim=9, axes=[0, 1, 2]))
    with pytest.raises(ValueError, match="at most 8 dimensions"):
        gp.grad_predict(np.zeros(5), np.zeros((4, 9)), return_var=True)


def test_x1_gradient_matvec_shape_checks():
    from george_b200 import kernels
    from george_b200._spec import DimensionMismatch
    k = kernels.ExpSquaredKernel(1.0, ndim=2).kernel
    x1, x2 = np.zeros((3, 2)), np.zeros((5, 2))
    for v in (np.zeros(4), np.zeros((5, 2)), np.zeros((3, 5)), np.zeros((5, 3, 1))):
        with pytest.raises(DimensionMismatch):
            k.x1_gradient_matvec(x1, x2, v)
    with pytest.raises(DimensionMismatch):
        k.x1_gradient_matvec(np.zeros((3, 1)), x2, np.zeros(5))


def test_without_device_raises():
    """No CPU fallback: with valid arguments and no H100 the contraction raises BGPError."""
    from george_b200 import _lib, kernels
    if _lib.load().bgp_device_count() > 0:
        pytest.skip("a GPU is present")
    k = kernels.ExpSquaredKernel(1.0, ndim=2).kernel
    for v in (np.zeros(5), np.zeros((5, 3))):
        with pytest.raises(_lib.BGPError):
            k.x1_gradient_matvec(np.zeros((3, 2)), np.zeros((5, 2)), v)
