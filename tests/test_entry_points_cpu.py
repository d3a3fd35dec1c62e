"""CPU: every Python entry point makes the same checks before it creates a handle (_B200Model._check_call) -- a FullSubNet_Plus
whose subband_num the reference forward runs, eval mode, a CUDA input -- so none of them can run a model the reference refuses."""
import pytest
import torch

from oracle import fsn_oracle as O

SUBBAND_ERR = "subband_num=2: the attention was built for 17 channels"


def _small(**kw):
    from fsnplus_b200.model import FullSubNet_Plus
    c = O.default_plus_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, fb_model_hidden_size=64)
    c.update(kw)
    return FullSubNet_Plus(**c)


@pytest.mark.parametrize("call", ["forward", "enhance_spectrum", "submit", "forward_host", "enhance_audio"])
def test_subband_num_refused_by_every_entry_point(call):
    """subband_num > 1 with an attention other than ECA: every entry point raises forward()'s error, instead of running the model as
    subband_num = 1 (what the handle's configuration says) or failing later for want of a device."""
    m = _small(channel_attention_model="SE", subband_num=2).eval()
    x = torch.zeros(1, 1, 33, 8)
    run = {"forward": lambda: m(x, x, x),
           "enhance_spectrum": lambda: m.enhance_spectrum(x, x, x),
           "submit": lambda: m.submit(x, x, x),
           "forward_host": lambda: m.forward_host(x, x, x),
           "enhance_audio": lambda: m.enhance_audio(torch.zeros(1, 256))}[call]
    with pytest.raises(RuntimeError, match=SUBBAND_ERR):
        run()
    assert m._handle is None


def test_forward_host_refuses_training_mode():
    m = _small()
    assert m.training
    x = torch.zeros(1, 1, 33, 8)
    with pytest.raises(NotImplementedError, match=r"\(eval\) forward only"):
        m.forward_host(x, x, x)
    assert m._handle is None
