"""CPU: serving.Engine's kv_cache_dtype argument is checked before any device work."""
import pytest
import torch

from aria_b200 import serving
from aria_b200.modeling_aria import AriaForConditionalGeneration
from aria_b200.serving import Engine


class _NoDevice:
    """Stand-in for the `ops` module: any kernel call is a test failure."""

    def __getattr__(self, name):
        raise AssertionError(f"device work ({name}) before the refusal")


class _StandInModel:
    """What Engine reads of a model before it allocates anything; any other attribute is a test failure."""

    _check_generate_args = staticmethod(AriaForConditionalGeneration._check_generate_args)

    def __init__(self):
        self.device = torch.device("cuda:0")

    def __getattr__(self, name):
        raise AssertionError(f"Engine read model.{name} before refusing the KV cache dtype")


@pytest.mark.parametrize("bad", ["fp16", "e4m3", "FP8", "", None, torch.float8_e4m3fn, 8])
def test_bad_kv_cache_dtype_is_refused_before_any_device_work(monkeypatch, bad):
    monkeypatch.setattr(serving, "ops", _NoDevice())
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        Engine(_StandInModel(), kv_cache_dtype=bad)


def test_the_default_is_bf16_pages():
    import inspect
    assert inspect.signature(Engine).parameters["kv_cache_dtype"].default == "bf16"
