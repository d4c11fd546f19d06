"""CPU restatement of the Stable Diffusion safety checker (stable_diffusion_pipeline.py:440-447: CLIPFeatureExtractor,
then diffusers' StableDiffusionSafetyChecker), for tests only.

preprocess : PIL bicubic resize of the shortest edge to 224 (long edge int(224 * long / short)), centre crop with
             top = (h - 224) // 2, left = (w - 224) // 2, then (u / 255 - mean) / std — what CLIPImageProcessorPil does.
vision_tower: CLIPVisionModel + post_layernorm on the CLS token + visual_projection, in float64.  `fp16_storage=True`
             rounds to fp16 where the native tower (csrc/sdw_safety.cu) stores fp16: the input pixels, the embeddings
             (patch conv + position embedding, one rounding), every LayerNorm output, every linear output (bias and
             residual before the one rounding), the attention output and the activation output.  The projection reads
             the fp16 pooled output and stays unrounded (the native one is fp32).
decide     : diffusers' per-image loop, literally, with the NumPy-1.x float64 promotion written out.
"""
import math

import numpy as np
import torch

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def resize_crop_u8(u8):
    """uint8 [H, W, 3] -> uint8 [224, 224, 3]: Pillow bicubic resize (shortest edge 224) and the centre crop"""
    from PIL import Image

    h, w = u8.shape[:2]
    if w <= h:
        nw, nh = 224, int(224 * h / w)
    else:
        nh, nw = 224, int(224 * w / h)
    r = np.asarray(Image.fromarray(np.ascontiguousarray(u8)).resize((nw, nh), Image.BICUBIC))
    top, left = (nh - 224) // 2, (nw - 224) // 2
    return r[top:top + 224, left:left + 224]


def preprocess(u8, mean=CLIP_MEAN, std=CLIP_STD):
    """uint8 [B, H, W, 3] -> float64 [B, 3, 224, 224] pixel values"""
    out = []
    for im in np.asarray(u8):
        c = resize_crop_u8(im).astype(np.float64) / 255.0
        out.append(((c - np.asarray(mean)) / np.asarray(std)).transpose(2, 0, 1))
    return torch.from_numpy(np.stack(out))


def _get(cfg, name):
    return cfg[name] if isinstance(cfg, dict) else getattr(cfg, name)


def vision_tower(pixels, sd, cfg, layers=None, fp16_storage=False, pooled_only=False):
    """pixels float [B, 3, 224, 224]; sd: a StableDiffusionSafetyChecker state dict (`vision_model.vision_model.*`,
    `visual_projection.weight`); cfg: CLIPVisionConfig fields.  Returns image_embeds float64 [B, proj] (or the pooled
    output with `pooled_only`)."""
    sd = {k: v.detach().to("cpu", torch.float64) for k, v in sd.items()}
    vm = "vision_model.vision_model."
    heads, H = _get(cfg, "num_attention_heads"), _get(cfg, "hidden_size")
    eps, act, p = _get(cfg, "layer_norm_eps"), _get(cfg, "hidden_act"), _get(cfg, "patch_size")
    n_layers = _get(cfg, "num_hidden_layers") if layers is None else layers
    d = H // heads

    def r(t):
        return t.half().double() if fp16_storage else t

    def ln(t, name):
        return r(torch.nn.functional.layer_norm(t, (H,), sd[name + ".weight"], sd[name + ".bias"], eps))

    def linear(t, name, resid=None):
        y = t @ sd[name + ".weight"].T + sd[name + ".bias"]
        return r(y if resid is None else y + resid)

    x = r(torch.as_tensor(pixels).double())
    B = x.shape[0]
    pe = torch.nn.functional.conv2d(x, sd[vm + "embeddings.patch_embedding.weight"], stride=p)
    pe = pe.flatten(2).transpose(1, 2)
    pos = sd[vm + "embeddings.position_embedding.weight"]
    cls = sd[vm + "embeddings.class_embedding"].expand(B, 1, H)
    x = r(torch.cat([cls, pe], dim=1) + pos)
    P = x.shape[1]
    x = ln(x, vm + "pre_layrnorm")
    for i in range(n_layers):
        pre = f"{vm}encoder.layers.{i}."
        h = ln(x, pre + "layer_norm1")
        q = linear(h, pre + "self_attn.q_proj").view(B, P, heads, d).transpose(1, 2)
        k = linear(h, pre + "self_attn.k_proj").view(B, P, heads, d).transpose(1, 2)
        v = linear(h, pre + "self_attn.v_proj").view(B, P, heads, d).transpose(1, 2)
        a = torch.softmax((q @ k.transpose(-1, -2)) / math.sqrt(d), dim=-1) @ v
        a = r(a.transpose(1, 2).reshape(B, P, H))
        x = linear(a, pre + "self_attn.out_proj", resid=x)
        h = ln(x, pre + "layer_norm2")
        f = linear(h, pre + "mlp.fc1")
        f = f * torch.sigmoid(1.702 * f) if act == "quick_gelu" else 0.5 * f * torch.erfc(-f / math.sqrt(2.0))
        x = linear(r(f), pre + "mlp.fc2", resid=x)
    pooled = ln(x[:, 0], vm + "post_layernorm")
    if pooled_only:
        return pooled
    return pooled @ sd["visual_projection.weight"].T


def cosines(image_embeds, sd):
    """fp32 [B, ns + nc] cosine similarities (special-care concepts first), computed in float64"""
    e = torch.as_tensor(image_embeds).double()
    E = torch.cat([sd["special_care_embeds"], sd["concept_embeds"]]).double()
    e, E = torch.nn.functional.normalize(e, dim=-1), torch.nn.functional.normalize(E, dim=-1)
    return (e @ E.T).float()


def decide(image_embeds, sd, cos=None):
    """diffusers' StableDiffusionSafetyChecker.forward decision loop for each image: (flags [B] bool, scores float64
    [B, ns + nc]).  `cos` (fp32 [B, ns + nc], special first) replaces the cosines computed from `image_embeds`."""
    if cos is None:
        cos = cosines(image_embeds, sd)
    cos = np.asarray(torch.as_tensor(cos).float().cpu().numpy())
    sw = [float(v) for v in torch.as_tensor(sd["special_care_embeds_weights"]).float()]
    cw = [float(v) for v in torch.as_tensor(sd["concept_embeds_weights"]).float()]
    ns = len(sw)
    flags, scores = [], np.zeros(cos.shape, dtype=np.float64)
    for i in range(cos.shape[0]):
        special_cos_dist, cos_dist = cos[i, :ns], cos[i, ns:]
        adjustment = 0.0
        bad_concepts = []
        for concept_idx in range(len(special_cos_dist)):
            concept_cos = np.float64(special_cos_dist[concept_idx])
            concept_threshold = np.float64(sw[concept_idx])
            s = np.round(concept_cos - concept_threshold + adjustment, 3)
            scores[i, concept_idx] = s
            if s > 0:
                adjustment = 0.01
        for concept_idx in range(len(cos_dist)):
            concept_cos = np.float64(cos_dist[concept_idx])
            concept_threshold = np.float64(cw[concept_idx])
            s = np.round(concept_cos - concept_threshold + adjustment, 3)
            scores[i, ns + concept_idx] = s
            if s > 0:
                bad_concepts.append(concept_idx)
        flags.append(len(bad_concepts) > 0)
    return np.asarray(flags), scores


# ---------------------------------------------------------------------------------------------------------------------
# fixtures shared by the CPU and GPU tests
# ---------------------------------------------------------------------------------------------------------------------
VISION = {
    "small": dict(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, image_size=224,
                  patch_size=32, hidden_act="quick_gelu", layer_norm_eps=1e-5),
    "ViT-L/14": dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                     image_size=224, patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5),
}


def hf_vision(kw, trained_like=False, seed=0, layers=None):
    """a transformers.CLIPVisionModel (fp32 holding fp16 values) and its config; `layers` cuts the tower"""
    from transformers import CLIPVisionConfig, CLIPVisionModel

    kw = dict(kw)
    if layers is not None:
        kw["num_hidden_layers"] = layers
    torch.manual_seed(seed)
    model = CLIPVisionModel(CLIPVisionConfig(**kw)).eval()
    with torch.no_grad():
        vm = model.vision_model
        H = kw["hidden_size"]
        if trained_like:
            # peaked attention (logit std ~ 4), a CLS sink, large residual channels at the CLS position and MLP
            # pre-activations reaching ~ -10, as in a trained tower
            vm.embeddings.class_embedding[[3, 77]] += torch.tensor([150.0, 250.0])
            for layer in vm.encoder.layers:
                at = layer.self_attn
                at.q_proj.weight.normal_(0.0, 2.0 / H ** 0.5)
                at.k_proj.weight.normal_(0.0, 2.0 / H ** 0.5)
                layer.mlp.fc1.weight.mul_(3.5)
            vm.embeddings.patch_embedding.weight.mul_(4.0)
        for n, p in model.named_parameters():
            if n.endswith("bias") or "layer_norm" in n or "layrnorm" in n:
                p.add_(torch.randn_like(p) * 0.05)
        for p in model.parameters():
            p.copy_(p.half().float())
    return model, model.config


def checker_state_dict(model, proj=768, ns=3, nc=17, seed=0):
    """diffusers-layout StableDiffusionSafetyChecker state dict around a CLIPVisionModel (fp16 values)"""
    g = torch.Generator().manual_seed(seed)
    sd = {"vision_model." + k: v.detach().clone() for k, v in model.state_dict().items()}
    H = model.config.hidden_size
    sd["visual_projection.weight"] = (torch.randn(proj, H, generator=g) / H ** 0.5).half().float()
    sd["concept_embeds"] = torch.randn(nc, proj, generator=g).half().float()
    sd["special_care_embeds"] = torch.randn(ns, proj, generator=g).half().float()
    sd["concept_embeds_weights"] = torch.full((nc,), 0.2).half().float()
    sd["special_care_embeds_weights"] = torch.full((ns,), 0.2).half().float()
    return sd


def test_frames(B, H, W, seed=0):
    """uint8 [B, H, W, 3]: smooth gradients, texture and a few hard edges, different per frame"""
    g = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    out = np.empty((B, H, W, 3), dtype=np.uint8)
    for b in range(B):
        f = np.stack([np.sin((c + 1 + b) * 3 * xx + yy * (2 + c)) for c in range(3)], -1) * 90 + 128
        f += g.normal(0, 25, (H, W, 3))
        f[H // 3: H // 2, W // 4: W // 2] = g.integers(0, 256, 3)
        out[b] = np.clip(f, 0, 255).astype(np.uint8)
    return out
