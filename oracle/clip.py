"""CPU restatement of `transformers.CLIPTextModel`'s forward (the text tower behind embed_text,
stable_diffusion_pipeline.py:809-820), for tests only.

x = tok[ids] + pos[p]; per layer (pre-LN): x += out_proj(attn(ln1(x))), x += fc2(act(fc1(ln2(x)))); y = final_ln(x).
Attention is causal with 64-wide heads: softmax(q k^T / sqrt(d)) v, key j visible to query i iff j <= i.
act: quick-GELU x sigmoid(1.702 x) ("quick_gelu", SD-1.x ViT-L/14) or erf GELU ("gelu", SD-2.x OpenCLIP-H).

Arithmetic is float64.  `fp16_storage=True` rounds to fp16 exactly where the native tower (csrc/sdw_clip.cu) stores fp16:
the embedding output, every LayerNorm output, every linear output (bias and residual added before the one rounding, as
the GEMM epilogue does), the attention output (probabilities unrounded) and the activation output.  It measures the
error an fp16-storage implementation is expected to have.
"""
import math

import torch


def _get(cfg, name):
    return cfg[name] if isinstance(cfg, dict) else getattr(cfg, name)


def text_model(ids, sd, cfg, layers=None, fp16_storage=False):
    """ids: integer [B, P]; sd: CLIPTextModel state dict; cfg: its config (object or dict with transformers' field names
    hidden_size, num_attention_heads, num_hidden_layers, hidden_act, layer_norm_eps).  `layers` < num_hidden_layers runs
    only the first layers (then the final LayerNorm).  Returns last_hidden_state float64 [B, P, hidden]."""
    sd = {k: v.detach().to("cpu", torch.float64) for k, v in sd.items()}
    heads = _get(cfg, "num_attention_heads")
    H = _get(cfg, "hidden_size")
    eps = _get(cfg, "layer_norm_eps")
    act = _get(cfg, "hidden_act")
    n_layers = _get(cfg, "num_hidden_layers") if layers is None else layers
    if act not in ("quick_gelu", "gelu"):
        raise ValueError(act)
    d = H // heads

    def r(t):
        return t.half().double() if fp16_storage else t

    def ln(t, name):
        return r(torch.nn.functional.layer_norm(t, (H,), sd[name + ".weight"], sd[name + ".bias"], eps))

    def linear(t, name, resid=None):
        y = t @ sd[name + ".weight"].T + sd[name + ".bias"]
        return r(y if resid is None else y + resid)

    ids = torch.as_tensor(ids).long().cpu()
    B, P = ids.shape
    x = r(sd["text_model.embeddings.token_embedding.weight"][ids] +
          sd["text_model.embeddings.position_embedding.weight"][:P])
    visible = torch.ones(P, P, dtype=torch.bool).tril()
    for i in range(n_layers):
        p = f"text_model.encoder.layers.{i}."
        h = ln(x, p + "layer_norm1")
        q = linear(h, p + "self_attn.q_proj").view(B, P, heads, d).transpose(1, 2)
        k = linear(h, p + "self_attn.k_proj").view(B, P, heads, d).transpose(1, 2)
        v = linear(h, p + "self_attn.v_proj").view(B, P, heads, d).transpose(1, 2)
        s = (q @ k.transpose(-1, -2)) / math.sqrt(d)
        a = torch.softmax(s.masked_fill(~visible, float("-inf")), dim=-1) @ v
        a = r(a.transpose(1, 2).reshape(B, P, H))
        x = linear(a, p + "self_attn.out_proj", resid=x)
        h = ln(x, p + "layer_norm2")
        f = linear(h, p + "mlp.fc1")
        if act == "quick_gelu":
            f = f * torch.sigmoid(1.702 * f)
        else:
            f = 0.5 * f * torch.erfc(-f / math.sqrt(2.0))
        x = linear(r(f), p + "mlp.fc2", resid=x)
    return ln(x, "text_model.final_layer_norm")
