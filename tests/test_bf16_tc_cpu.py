"""The tc_precision setting is validated before any device work: an unknown value, or bf16 on a model without tensor
cores, raises ValueError from Model and from PipelinedCodec.  Runs without a GPU."""
import types

import pytest

from bitswap_b200.codec import PipelinedCodec
from bitswap_b200.config import preset
from bitswap_b200.model import Model


@pytest.mark.parametrize("kw,match", [({"use_tensor_cores": False, "tc_precision": "bf16"}, "use_tensor_cores=True"),
                                      ({"use_tensor_cores": True, "tc_precision": "fp8"}, "tc_precision must be one of"),
                                      ({"use_tensor_cores": True, "tc_precision": None}, "tc_precision must be one of")])
def test_model_refuses_before_device_work(kw, match):
    with pytest.raises(ValueError, match=match):
        Model.from_config(preset("tiny3"), max_batch=1, **kw)


def test_pipelined_codec_refuses_bf16_without_tensor_cores():
    bins = types.SimpleNamespace(device=0)        # never touched: the first lane's Model refuses first
    with pytest.raises(ValueError, match="use_tensor_cores=True"):
        PipelinedCodec(preset("tiny3"), {}, bins, 4, use_tensor_cores=False, tc_precision="bf16")
