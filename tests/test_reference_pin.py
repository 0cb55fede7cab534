"""Pins the oracle restatement of the reference's own code (oracle/models_ref.py <- the reference's models.py) to the REAL file:
models.py is imported unmodified (tests/golden/reference_import.py stands in for the ten `diffusers` names it imports) and run next
to the restatement on the same weights and inputs - every shipped config's hint encoder, every processor class (plain / v1 / V2 /
post_add / concat_hidden / stacked chains / scale != 1), and a whole tiny UNet with the reference's processors installed.
Where the reference tree is present the reference runs live; elsewhere its committed results take over (tests/golden/reference_pin.pt
from tests/golden/make_reference_pin_golden.py for these cases, tests/golden/reference_models.pt from
tests/golden/make_reference_golden.py for the front-half vectors that the CUDA path is also checked against under `-m gpu`)."""
import functools
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from oracle import models_ref as MR  # noqa: E402
from tests.golden import make_reference_pin_golden as P  # noqa: E402
from tests.golden import reference_import as RI  # noqa: E402

@pytest.fixture(autouse=True)
def _single_thread():
    """fp32 summation order of the CPU convolutions depends on the thread count / scheduling; the comparisons below are between two
    programs that issue the same torch calls, so one thread makes them reproducible to the last few ulps."""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


needs_reference = pytest.mark.skipif(not RI.available(), reason="the reference tree is not present on this machine")
CONFIGS = P.CONFIGS


@functools.lru_cache(maxsize=1)
def _gold():
    return P.load()


def _pair(kind, key, run, *args):
    """(reference, restatement) results of one case.  Where the reference tree exists both run live and whole tensors are
    compared; elsewhere the restatement is compared with the committed reference results (tests/golden/reference_pin.pt,
    written by the same program), on the fixed seeded sample of each tensor stored there."""
    if RI.available():
        with P.full_tensors():
            return run(RI.reference_models(), *args), run(MR, *args)
    return _gold()[kind][key], run(MR, *args)


def _close(o, r, rtol, atol, what):
    assert o["shape"] == r["shape"], what
    assert abs(o["amax"] - r["amax"]) <= rtol * r["amax"] + atol, what
    assert o["s"].shape == r["s"].shape, what
    if r["s"].numel():
        assert float((o["s"] - r["s"]).abs().max()) <= rtol * r["amax"] + atol, what


@pytest.mark.parametrize("name", CONFIGS)
def test_hint_encoder_restatement_equals_the_reference(name):
    """ControlLoRA.__init__ wiring + forward (models.py:618-835) for every shipped configs/*.json: same state-dict keys / shapes,
    and - on the same weights - bit-comparable control states and parameter gradients."""
    cfg = RI.reference_config(name) if RI.available() else _gold()["configs"][name]
    ref, ora = _pair("hint", name, P.run_hint, cfg)
    assert ora["keys"] == ref["keys"]
    assert ora["types"] == ref["types"] and ora["attrs"] == ref["attrs"]
    assert len(ora["states"]) == len(ref["states"])
    for a, b in zip(ora["states"], ref["states"]):
        _close(a, b, 1e-4, 0.0, "control state")
    assert list(ora["grads"]) == list(ref["grads"])
    for n, b in ref["grads"].items():
        if b is None:
            assert ora["grads"][n] is None, n
        else:
            _close(ora["grads"][n], b, 1e-3, 1e-9, n)
    # the processors received the same injected tensors (models.py:826-829)
    assert all(all(lvl) for lvl in ref["injected"]) and ora["injected"] == ref["injected"]


@pytest.mark.parametrize("case", list(P.PROC_CASES))
def test_processor_restatement_equals_the_reference(case):
    """One processor call (models.py:118-152 / 222-287 / 357-431) on the same attention module, hidden states, text states and
    control states: output, d hidden, every parameter gradient, d control - reference code vs restatement."""
    ref, ora = _pair("processor", case, P.run_processor, case)
    _close(ora["y"], ref["y"], 2e-5, 1e-8, "output")
    _close(ora["dh"], ref["dh"], 2e-5, 1e-8, "d hidden")
    assert set(ora["grads"]) == set(ref["grads"])
    for n in ref["grads"]:
        _close(ora["grads"][n], ref["grads"][n], 2e-5, 1e-8, n)
    assert len(ora["dc"]) == len(ref["dc"]) and (len(ref["dc"]) > 0) == ref["has_control"]
    for a, b in zip(ora["dc"], ref["dc"]):
        _close(a, b, 2e-5, 1e-8, "d control")


@pytest.mark.parametrize("variant", P.UNET_VARIANTS)
def test_unet_with_reference_processors_equals_unet_with_restated_processors(variant):
    """The whole training-step front half on a tiny SD-style UNet (the UNet restatement is the same on both sides): the reference's
    ControlLoRA + processors + the wiring of train_text_to_image_control_lora.py:469-487 against oracle/models_ref.py."""
    ref, ora = _pair("unet", variant, P.run_unet, variant)
    _close(ora["pred"], ref["pred"], 2e-5, 0.0, "pred")
    assert abs(ora["loss"] - ref["loss"]) <= 1e-6 * abs(ref["loss"])
    assert set(ora["grads"]) == set(ref["grads"]) and len(ref["grads"]) > 50
    for n in ref["grads"]:
        _close(ora["grads"][n], ref["grads"][n], 1e-4, 1e-9, n)


@pytest.mark.parametrize("case", ["v1_stacked", "v2", "post_add", "concat"])
def test_oracle_matches_the_golden_vectors_generated_by_the_reference(case):
    """Runs everywhere (no reference tree needed): the committed vectors were computed by the reference's own models.py
    (tests/golden/make_reference_golden.py); the restatement must reproduce them from the same seeded weights and inputs."""
    from tests.golden import make_reference_golden as G

    gold = torch.load(G.OUT, weights_only=False)[case]
    got = G.run_front_half(MR, case)
    close = lambda a, b: float((a - b).abs().max()) <= 2e-5 * float(b.abs().max()) + 1e-9
    assert close(got["pred"], gold["pred"]) and close(got["loss"], gold["loss"]) and close(got["state_norms"], gold["state_norms"])
    assert all(close(a, b) for a, b in zip(got["states"], gold["states"]))
    assert got["grads"]["names"] == gold["grads"]["names"] and got["grad_norms"]["names"] == gold["grad_norms"]["names"]
    assert close(got["grads"]["flat"], gold["grads"]["flat"]) and close(got["grads"]["norms"], gold["grads"]["norms"])
    assert float(((got["grad_norms"]["values"] - gold["grad_norms"]["values"]).abs() / gold["grad_norms"]["values"].clamp_min(1e-12)).max()) < 1e-3


@needs_reference
def test_committed_golden_vectors_are_what_the_reference_computes_now():
    """Guards the fixture itself: regenerating one case from the reference's models.py gives the committed numbers."""
    from tests.golden import make_reference_golden as G

    gold = torch.load(G.OUT, weights_only=False)["v2"]
    now = G.run_front_half(RI.reference_models(), "v2")
    assert float((now["pred"] - gold["pred"]).abs().max()) <= 1e-6 * float(gold["pred"].abs().max())
    assert float((now["grads"]["flat"] - gold["grads"]["flat"]).abs().max()) <= 1e-5 * float(gold["grads"]["flat"].abs().max())


@needs_reference
def test_committed_pin_results_are_what_the_reference_computes_now():
    """Guards tests/golden/reference_pin.pt: regenerating one case of each kind from the reference's models.py gives the
    committed samples."""
    gold = _gold()
    name = "diffusiondb-canny-v2"
    now = {"hint": P.run_hint(RI.reference_models(), gold["configs"][name]),
           "processor": P.run_processor(RI.reference_models(), "v2_stacked_control"),
           "unet": P.run_unet(RI.reference_models(), "v2")}
    for kind, key in (("hint", name), ("processor", "v2_stacked_control"), ("unet", "v2")):
        g, n = gold[kind][key], now[kind]
        leaves = []

        def walk(a, b):
            if isinstance(b, dict) and "s" in b:
                leaves.append((a, b))
            elif isinstance(b, dict):
                assert set(a) == set(b)
                for k in b:
                    walk(a[k], b[k])
            elif isinstance(b, list):
                assert len(a) == len(b)
                for x, y in zip(a, b):
                    walk(x, y)
            else:
                assert a == b
        walk(n, g)
        assert leaves
        for a, b in leaves:
            _close(a, b, 1e-6, 1e-12, kind)
