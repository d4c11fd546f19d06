"""CLIP text-tower fixtures shared by the CPU oracle pin (test_clip_cpu.py) and the native tower tests (test_clip_gpu.py):
the three tower configurations and `transformers.CLIPTextModel`s with fp16-rounded weights, either as initialised or
rescaled to look like a trained tower."""
import torch
import torch.nn.functional as Fn

CONFIGS = {
    "small": dict(vocab_size=1000, hidden_size=256, intermediate_size=1024, num_hidden_layers=3, num_attention_heads=4,
                  max_position_embeddings=77, hidden_act="quick_gelu"),
    "sd1x-ViT-L": dict(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                       num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu"),
    "sd2x-OpenCLIP-H-23": dict(vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=23,
                               num_attention_heads=16, max_position_embeddings=77, hidden_act="gelu"),
}

# residual channels that carry 150..300 at position 0 in the trained-like weights (all below the smallest width, 256)
BIG_CHANNELS = (3, 77, 150)
BIG_VALUES = (150.0, 220.0, 300.0)


def _trained_like_(model):
    """Rescale HF's init so that the tower behaves like a trained CLIP: peaked attention rows (q / k weights with
    logit std ~ 4), a sink at the BOS position (each layer's q bias points at position 0's key), a few residual
    channels of magnitude 150..300 at position 0 (LayerNorm rows with a large mean and spread), and MLP
    pre-activations reaching ~ -10 (the negative tail of the activation)."""
    c = model.config
    H, heads = c.hidden_size, c.num_attention_heads
    tm = model.text_model
    pos = tm.embeddings.position_embedding.weight
    pos[0, list(BIG_CHANNELS)] += torch.tensor(BIG_VALUES)
    for layer in tm.encoder.layers:
        at = layer.self_attn
        # LayerNorm output has unit variance per channel: q / k components of std 2, logits q.k / 8 of std ~ 4
        at.q_proj.weight.normal_(0.0, 2.0 / H ** 0.5)
        at.k_proj.weight.normal_(0.0, 2.0 / H ** 0.5)
        u = Fn.layer_norm(pos[:1], (H,), layer.layer_norm1.weight, layer.layer_norm1.bias, c.layer_norm_eps)
        k0 = at.k_proj(u).view(heads, -1)
        # |k0| ~ 16 per head: a q bias of norm 3 along it lifts key 0 by ~ 6 logits for every query
        at.q_proj.bias.copy_((3.0 * k0 / k0.norm(dim=1, keepdim=True)).flatten())
        layer.mlp.fc1.weight.mul_(3.5)


def hf_model(cfg_kw, trained_like=False, seed=0):
    """a transformers.CLIPTextModel in fp32 whose parameters are fp16 values (what the native tower is handed)."""
    from transformers import CLIPTextConfig, CLIPTextModel

    torch.manual_seed(seed)
    model = CLIPTextModel(CLIPTextConfig(**cfg_kw)).eval()
    with torch.no_grad():
        if trained_like:
            _trained_like_(model)
        for p in model.parameters():
            p.copy_(p.half().float())
        # random-init LayerNorm affines / biases are 1 / 0: perturb them so that every parameter is exercised
        for n, p in model.named_parameters():
            if n.endswith("bias") or "layer_norm" in n:
                p.add_((torch.randn_like(p) * 0.05).half().float())
    return model


def prompt_ids(vocab, B, seed=1):
    """[B, 77] token ids: a BOS-like first token, random tokens, and one padded prompt (EOS repeated to the end)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, vocab, (B, 77), generator=g)
    ids[:, 0] = vocab - 2
    ids[0, 20:] = vocab - 1
    return ids
