# -*- coding: utf-8 -*-
"""tools/hodlr_phase_profile.py without a device: argument parsing, kernel names and the cutting of a trace into
up-sweep and solve windows, on a synthetic chrome trace."""
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


def _step(t):
    """One compute + dot_solve on the GPU timeline, starting at t (us)."""
    return [
        _ev("Memcpy DtoD (Device -> Device)", t, 2, "gpu_memcpy"),      # compute's copy of x: not a solve
        _ev("void bgp::a2_eval_kernel<1>(bgp::A2Args)", t + 10, 50),
        _ev("Memcpy HtoD (Pageable -> Device)", t + 70, 1, "gpu_memcpy"),
        _ev("void bgp::finalize_panels_kernel(bgp::NodeDesc const*, bgp::PanelTile const*, double*, long, double*, long)",
            t + 80, 10),
        _ev("void bgp::leaf_solve_kernel<8>(bgp::LeafDesc const*, double const*, double*, long, int const*, int, int, int)",
            t + 95, 100),
        _ev("Memset (Device)", t + 200, 1, "gpu_memset"),
        _ev("void bgp::gram_tn_small_kernel<4>(bgp::NodeDesc const*, double const*, long, double const*, long, int, "
            "double*, long)", t + 203, 7),
        _ev("void bgp::small_solve_kernel(bgp::NodeDesc const*, double*, long, int, int, int, double*, double*, int)",
            t + 212, 5),
        _ev("void bgp::update_nn_kernel(bgp::NodeDesc const*, double const*, long, double*, long, int, int, "
            "double const*, long, int)", t + 220, 10),
        _ev("Memcpy DtoH (Device -> Pageable)", t + 235, 1, "gpu_memcpy"),
        _ev("Memcpy DtoD (Device -> Device)", t + 300, 2, "gpu_memcpy"),
        _ev("void bgp::leaf_solve_kernel<1>(bgp::LeafDesc const*, double const*, double*, long, int const*, int, int, int)",
            t + 305, 20),
        _ev("void bgp::gram_tn_kernel(bgp::NodeDesc const*, double const*, long, double const*, long, int, double*, long)",
            t + 330, 5),
        _ev("void bgp::dot_kernel(double const*, double const*, long, double*)", t + 340, 3),
        _ev("Memcpy DtoH (Device -> Pageable)", t + 345, 1, "gpu_memcpy"),
    ]


def test_kernel_keys(prof):
    assert prof.kernel_key("void bgp::leaf_solve_kernel<8>(bgp::LeafDesc const*)", "kernel") == "leaf_solve<8>"
    assert prof.kernel_key("void bgp::gram_tn_small_kernel<2>(int)", "kernel") == "gram_tn_small<2>"
    assert prof.kernel_key("void bgp::finalize_panels_kernel(int)", "kernel") == "finalize_panels"
    assert prof.kernel_key("Memset (Device)", "gpu_memset") == "memset"
    assert prof.kernel_key("Memcpy DtoH (Device -> Pinned)", "gpu_memcpy") == "memcpy_DtoH"


def test_windows_and_idle_time(prof):
    trace = {"traceEvents": _step(0) + _step(1000) + [{"ph": "X", "cat": "cpu_op", "name": "x", "ts": 5, "dur": 1}]}
    s = prof.summarise(prof.gpu_activities(trace))
    up, so = s["upsweep"], s["solve"]
    assert up["steps"] == 2 and so["steps"] == 2
    # up-sweep: 80 .. 230 us, busy 10 + 100 + 1 + 7 + 5 + 10 = 133 us
    assert up["span_ms"] == pytest.approx(0.150)
    assert up["busy_ms"] == pytest.approx(0.133)
    assert up["idle_ms"] == pytest.approx(0.017)
    assert list(up["kernels"]) == ["leaf_solve<8>", "finalize_panels", "update_nn", "gram_tn_small<4>", "small_solve",
                                   "memset"]
    assert up["kernels"]["leaf_solve<8>"] == {"ms": pytest.approx(0.1), "launches": 1.0}
    # solve: 300 .. 343 us, busy 2 + 20 + 5 + 3 = 30 us
    assert so["span_ms"] == pytest.approx(0.043)
    assert so["idle_ms"] == pytest.approx(0.013)
    assert set(so["kernels"]) == {"memcpy_DtoD", "leaf_solve<1>", "gram_tn", "dot"}
    text = prof.format_summary(s, "hdr")
    assert text.startswith("hdr\nupsweep: span 0.150 ms/step")


def test_argument_parsing(prof):
    a = prof.parse_args(["--out", "o"])
    assert a.out == "o" and a.workload == "cfg3" and a.steps == 3 and a.warmup == 2 and a.exhaust == "lowrank"
    assert os.path.samefile(a.root, ROOT)
    with pytest.raises(SystemExit):
        prof.parse_args([])
