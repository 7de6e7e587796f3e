# -*- coding: utf-8 -*-
"""tools/hodlr_phase_profile.py without a device: the factor window (leaf factorisation beside the ACA loop) of a
synthetic chrome trace."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def prof():
    spec = importlib.util.spec_from_file_location("hodlr_phase_profile", os.path.join(ROOT, "tools", "hodlr_phase_profile.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _ev(name, ts, dur, cat="kernel"):
    return {"ph": "X", "cat": cat, "name": name, "ts": ts, "dur": dur}


def _compute(t, leaf="void bgp::leaf_factor_kernel<2>(bgp::DevProgram const*, double const*)"):
    """The factorisation part of one compute() on the GPU timeline, starting at t (us): leaves on one stream, the ACA
    loop on the other, then the up-sweep."""
    return [
        _ev("Memcpy DtoD (Device -> Device)", t, 2, "gpu_memcpy"),
        _ev(leaf, t + 10, 400),
        _ev("Memcpy HtoD (Pageable -> Device)", t + 20, 1, "gpu_memcpy"),
        _ev("void bgp::a2_init_kernel(bgp::A2Args)", t + 300, 50),
        _ev("void bgp::a2_eval_kernel<2, 3>(bgp::A2Args)", t + 420, 30),
        _ev("void bgp::a2_decide_kernel(bgp::A2Args)", t + 455, 20),
        _ev("void bgp::a2_tick_kernel(int*, int const*, unsigned long long, int)", t + 480, 2),
        _ev("void bgp::a2_eval_kernel<2, 3>(bgp::A2Args)", t + 490, 30),
        _ev("void bgp::a2_tick_kernel(int*, int const*, unsigned long long, int)", t + 530, 2),
        _ev("Memcpy DtoH (Device -> Pageable)", t + 540, 1, "gpu_memcpy"),  # iteration count: after the last tick
        _ev("void bgp::finalize_panels_kernel(bgp::NodeDesc const*)", t + 600, 10),
        _ev("void bgp::leaf_solve_kernel<8>(bgp::LeafDesc const*)", t + 615, 20),
        _ev("Memcpy DtoH (Device -> Pageable)", t + 640, 1, "gpu_memcpy"),
    ]


def test_factor_window(prof):
    trace = {"traceEvents": _compute(0) + _compute(2000)}
    s = prof.summarise(prof.gpu_activities(trace))
    f = s["factor"]
    assert f["steps"] == 2 and s["upsweep"]["steps"] == 2
    # 10 .. 532 us; busy: leaf 10..410 with the copy and a2_init inside, then 420..450, 455..475, 480..482, 490..520,
    # 530..532
    assert f["span_ms"] == pytest.approx(0.522)
    assert f["busy_ms"] == pytest.approx(0.400 + 0.030 + 0.020 + 0.002 + 0.030 + 0.002)
    assert f["idle_ms"] == pytest.approx(0.522 - 0.484)
    assert f["leaf_ms"] == pytest.approx(0.400)
    assert f["a2_init_start_ms"] == pytest.approx(0.290)
    # a2_init 300..350, then the loop kernels: 50 + 30 + 20 + 2 + 30 + 2
    assert f["aca_busy_ms"] == pytest.approx(0.134)
    assert f["kernels"]["a2_tick"]["launches"] == 2.0
    assert "memcpy_DtoH" not in f["kernels"] and "finalize_panels" not in f["kernels"]
    assert f["kernels"]["leaf_factor<2>"] == {"ms": pytest.approx(0.4), "launches": 1.0}
    text = prof.format_summary(s, "hdr")
    assert text.startswith("hdr\nfactor: span 0.522 ms/step")
    assert "leaf kernel span 0.400 ms, a2_init starts at +0.290 ms, ACA kernels busy 0.134 ms" in text


def test_factor_window_of_the_generic_leaf_kernel(prof):
    leaf = "void bgp::leaf_build_factor_kernel(bgp::DevProgram const*, double const*)"
    s = prof.summarise(prof.gpu_activities({"traceEvents": _compute(0, leaf)}))
    assert s["factor"]["leaf_ms"] == pytest.approx(0.400)
    assert list(s["factor"]["kernels"])[0] == "leaf_build_factor"


def test_trace_without_a_factorisation_has_no_factor_window(prof):
    s = prof.summarise(prof.gpu_activities({"traceEvents": _compute(0)[-3:]}))
    assert "factor" not in s and s["upsweep"]["steps"] == 1
    assert prof.format_summary(s, "hdr").startswith("hdr\nupsweep: ")
