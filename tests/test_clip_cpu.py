"""The CLIP oracle (oracle/clip.py) pinned to the installed transformers.CLIPTextModel: in float64 on the same weights
the two must agree to rounding, for the three tower configurations, with HF's init and with the trained-like weights.
No GPU."""
import pytest
import torch

from _clip_fixtures import CONFIGS, hf_model, prompt_ids
from oracle.clip import text_model


@pytest.mark.parametrize("trained_like", [False, True], ids=["hf-init", "trained-like"])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_oracle_matches_transformers_fp64(name, trained_like):
    cfg_kw = CONFIGS[name]
    model = hf_model(cfg_kw, trained_like)
    ids = prompt_ids(cfg_kw["vocab_size"], 2)
    with torch.no_grad():
        got = text_model(ids, model.state_dict(), model.config)
        ref = model.double()(ids)[0]
    rel = float((got - ref).norm() / ref.norm())
    err = float((got - ref).abs().max())
    assert rel <= 1e-9 and err <= 1e-9 * float(ref.abs().max()), (name, rel, err)


def test_trained_like_weights_are_peaked_and_stay_finite_in_fp16():
    """the fixture does what it claims on ViT-L: layer 0's attention logits have std ~ 4 and a BOS sink, position 0
    carries residual channels of 150..300, the first MLP's pre-activations reach ~ -10; the fp16-storage oracle is
    finite."""
    import torch.nn.functional as Fn

    cfg_kw = CONFIGS["sd1x-ViT-L"]
    model = hf_model(cfg_kw, trained_like=True)
    sd = {k: v.double() for k, v in model.state_dict().items()}
    ids = prompt_ids(cfg_kw["vocab_size"], 2)
    p = "text_model.encoder.layers.0."
    x = sd["text_model.embeddings.token_embedding.weight"][ids] + sd["text_model.embeddings.position_embedding.weight"][:77]
    assert float(x[:, 0].abs().max()) >= 150
    h = Fn.layer_norm(x, (768,), sd[p + "layer_norm1.weight"], sd[p + "layer_norm1.bias"], 1e-5)
    q = (h @ sd[p + "self_attn.q_proj.weight"].T + sd[p + "self_attn.q_proj.bias"]).view(2, 77, 12, 64).transpose(1, 2)
    k = (h @ sd[p + "self_attn.k_proj.weight"].T + sd[p + "self_attn.k_proj.bias"]).view(2, 77, 12, 64).transpose(1, 2)
    s = q @ k.transpose(-1, -2) / 8
    free = s[..., 1:, 1:].tril()  # the logits of visible keys other than the sink
    free = free[free != 0]
    assert 3.0 <= float(free.std()) <= 6.0, float(free.std())
    sink = s[..., 1:, 0] - s[..., 1:, 1:].mean(-1)
    assert float(sink.mean()) >= 4.0, float(sink.mean())
    f = h @ sd[p + "mlp.fc1.weight"].T  # fc1 on a unit-variance LayerNorm output
    assert float(f.min()) <= -8.0, float(f.min())
    with torch.no_grad():
        y = text_model(ids, model.state_dict(), model.config, fp16_storage=True)
    assert bool(torch.isfinite(y).all())
