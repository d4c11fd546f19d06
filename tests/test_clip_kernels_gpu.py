"""The CLIP text tower's own kernels (csrc/sdw_clip.cu), each called through the C ABI and compared with a float64
reference of the same operation on the same fp16 inputs: the token + position embedding gather (bit for bit), the
77 x 77 causal attention per head (peaked rows, a sink, a diagonal, exact causality), quick-GELU / erf GELU over every
finite fp16 value, and the tower's linear layers on the GEMM kernel at the shapes the tower runs.

Outputs start as NaN; the bytes after every written view start as a sentinel and must come back unchanged; the inputs
must be unchanged afterwards."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

SENT = -7.25  # sentinel of the bytes after an output view
TAIL = 4096   # sentinel elements after each output


def _n():
    from stable_diffusion_videos_b200 import _native as n
    return n


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _out(numel, tail=TAIL):
    """a NaN output of `numel` fp16 values followed by `tail` sentinels; returns (buffer, view)."""
    buf = torch.full((numel + tail,), SENT, dtype=torch.float16, device="cuda")
    buf[:numel] = float("nan")
    return buf, buf[:numel]


def _tail_ok(buf, numel):
    return bool((buf[numel:] == SENT).all())


# ----------------------------------------------------------------------------------------------------------------------
# embedding: x[r] = fp16(tok[clamp(ids[r])] + pos[r % P]), bit for bit
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [256, 768, 1024])
@pytest.mark.parametrize("P", [1, 31, 32, 33, 77, 96])
def test_clip_embed_bit_exact(P, H):
    n = _n()
    vocab = 1000
    g = _gen(P * 7 + H)
    tok = (torch.randn(vocab, H, generator=g) * 0.5).half().cuda()
    pos = (torch.randn(P, H, generator=g) * 0.5).half().cuda()
    for rows in sorted({P, min(8 * P, 8 * 77)}):
        ids = torch.randint(0, vocab, (rows,), generator=g, dtype=torch.int32)
        edge = torch.tensor([0, vocab - 1, -1, vocab + 5, -2 ** 31, 2 ** 31 - 1], dtype=torch.int32)
        k = min(rows, edge.numel())
        ids[-k:] = edge[:k]  # edge ids last, so that P = 1 (one row per prompt) still sees the vocabulary ends
        ids = ids.cuda()
        before = (ids.clone(), tok.clone(), pos.clone())
        buf, x = _out(rows * H)
        n.clip_embed(ids, tok, pos, rows, P, x)
        torch.cuda.synchronize()
        r = torch.arange(rows, device="cuda")
        ref = (tok.float()[ids.long().clamp(0, vocab - 1)] + pos.float()[r % P]).half()
        assert torch.equal(x.view(rows, H).view(torch.int16), ref.view(torch.int16)), (P, H, rows)
        assert _tail_ok(buf, rows * H)
        assert all(torch.equal(a, b) for a, b in zip(before, (ids, tok, pos)))


# ----------------------------------------------------------------------------------------------------------------------
# causal attention per (sample, head)
# ----------------------------------------------------------------------------------------------------------------------
def _attn_ref64(qkv, B, P, heads):
    """float64 causal attention of fp16 qkv [B][P][3H] -> ([B][P][H], max|v| per (sample, head column) [B][1][H])."""
    H = 64 * heads
    x = qkv.double().view(B, P, 3, heads, 64)
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))  # [B][heads][P][64]
    s = (q @ k.transpose(-1, -2)) * 0.125
    s = s.masked_fill(~torch.ones(P, P, dtype=torch.bool, device=qkv.device).tril(), float("-inf"))
    p = torch.softmax(s, dim=-1)
    out = (p @ v).transpose(1, 2).reshape(B, P, H)
    vmax = v.abs().amax(dim=2).reshape(B, 1, H)
    return out, vmax, p


def _attn_inputs(kind, B, P, heads, seed):
    """fp16 qkv [B][P][3H] whose logits have std ~ 5 ('peaked'), whose key 0 wins every row by > 25 logits ('sink'),
    or whose key i wins row i ('diag')."""
    g = _gen(seed)
    q = torch.randn(B, P, heads, 64, generator=g)
    k = torch.randn(B, P, heads, 64, generator=g)
    v = torch.randn(B, P, heads, 64, generator=g)
    if kind == "peaked":
        q, k = q * 2.2, k * 2.2  # logit = q.k / 8: std 2.2^2 = 4.8
    elif kind == "sink":
        q[..., 0] = 8.0
        k[:, 0, :, 0] = 50.0     # key 0: + 50 logits; every other key: std ~ 1.4
    elif kind == "diag":
        k = k * 1.5
        q = k.clone()            # logit(i, i) = |k_i|^2 / 8 ~ 18, logit(i, j != i) std ~ 2.3
    else:
        raise ValueError(kind)
    return torch.stack([q, k, v], dim=2).reshape(B, P, 3 * heads * 64).half().cuda()


def _attn_case(kind, B, P, heads, seed=0):
    """run one case; returns (worst err / bound, reference probabilities, output)."""
    n = _n()
    H = 64 * heads
    qkv = _attn_inputs(kind, B, P, heads, seed)
    before = qkv.clone()
    buf, out = _out(B * P * H)
    n.clip_attention(qkv, B, P, heads, out)
    torch.cuda.synchronize()
    assert torch.equal(qkv, before)
    assert _tail_ok(buf, B * P * H)
    ref, vmax, p = _attn_ref64(qkv, B, P, heads)
    o = out.view(B, P, H).double()
    assert bool(torch.isfinite(o).all())
    bound = 2.0 ** -10 * ref.abs() + 2.0 ** -12 * vmax
    return float(((o - ref).abs() / bound).max()), p, o


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("heads", [1, 4, 12, 16])
@pytest.mark.parametrize("P", [1, 2, 31, 32, 33, 63, 64, 65, 77, 95, 96])
def test_clip_attention_peaked(P, heads, B):
    # |out - ref| <= 2^-10 |ref| + 2^-12 max|v| per element: the fp16 output rounding (2^-11 relative) with 2x room,
    # plus __expf and the fp32 sums; the worst ratio measured on an H100 is recorded in the commit that added this test
    ratio, _, _ = _attn_case("peaked", B, P, heads, seed=P * 100 + heads * 10 + B)
    assert ratio <= 1.0, ratio


@pytest.mark.parametrize("kind", ["sink", "diag"])
@pytest.mark.parametrize("P", [1, 2, 31, 32, 33, 63, 64, 65, 77, 95, 96])
def test_clip_attention_sink_and_diagonal(P, kind):
    ratio, p, o = _attn_case(kind, 3, P, 4, seed=P)
    win = p.argmax(dim=-1)
    rows = torch.arange(P, device=p.device)
    if kind == "sink":
        assert bool((win == 0).all())
        top2 = p.topk(min(2, P), dim=-1).values
        if P > 1:  # the runner-up carries less than e^-25 of the winner's weight
            assert float((top2[..., 1] / top2[..., 0]).max()) < math.exp(-25)
    else:
        assert bool((win == rows).all())
    assert ratio <= 1.0, (kind, ratio)


@pytest.mark.parametrize("r0", [1, 32, 64, 76])
def test_clip_attention_causality_exact(r0):
    """poisoning Q, K and V of every row >= r0 with NaN leaves rows < r0 finite and bit-identical: a query never reads
    a later key or value.  NaN only enters arithmetic; no address depends on it."""
    n = _n()
    B, P, heads = 2, 77, 12
    H = 64 * heads
    qkv = _attn_inputs("peaked", B, P, heads, seed=5)
    outs = []
    for poison in (False, True):
        x = qkv.clone()
        if poison:
            x[:, r0:] = float("nan")
        buf, out = _out(B * P * H)
        n.clip_attention(x, B, P, heads, out)
        torch.cuda.synchronize()
        assert _tail_ok(buf, B * P * H)
        outs.append(out.view(B, P, H).clone())
    clean, poisoned = outs
    assert bool(torch.isfinite(poisoned[:, :r0]).all())
    assert torch.equal(poisoned[:, :r0].view(torch.int16), clean[:, :r0].view(torch.int16))
    assert bool(torch.isnan(poisoned[:, r0:]).all())


# ----------------------------------------------------------------------------------------------------------------------
# activations over every finite fp16 value
# ----------------------------------------------------------------------------------------------------------------------
def _ordered(h):
    """fp16 bit patterns -> integers in value order (+0 and -0 both 0): adjacent fp16 values differ by 1."""
    i = h.view(torch.int16).to(torch.int32)
    return torch.where(i < 0, -(i & 0x7FFF), i)


@pytest.mark.parametrize("gelu_erf", [0, 1], ids=["quick_gelu", "gelu"])
def test_clip_act_every_fp16_value(gelu_erf):
    """the 63 488 finite fp16 values are exactly 248 blocks of 256 threads: one more value makes a ragged last block.
    Every result lies within one fp16 ulp of the float64 result rounded to fp16."""
    n = _n()
    bits = torch.arange(-2 ** 15, 2 ** 15, dtype=torch.int32).to(torch.int16)
    vals = bits.view(torch.float16)
    vals = vals[torch.isfinite(vals)]
    assert vals.numel() == 63488
    vals = torch.cat([vals, torch.tensor([1.5], dtype=torch.float16)])
    N = vals.numel()
    buf = torch.full((N + TAIL,), SENT, dtype=torch.float16, device="cuda")
    buf[:N] = vals.cuda()
    n.clip_act(buf, N, gelu_erf)
    torch.cuda.synchronize()
    assert _tail_ok(buf, N)
    v = vals.double()
    ref = 0.5 * v * torch.erfc(-v / math.sqrt(2.0)) if gelu_erf else v * torch.sigmoid(1.702 * v)
    ref16 = ref.half()
    got = buf[:N].cpu()
    d = (_ordered(got) - _ordered(ref16)).abs()
    worst = int(d.argmax())
    print(f"clip_act gelu_erf={gelu_erf}: {int((d > 0).sum())} of {N} results not the rounded float64 value")
    assert int(d.max()) <= 1, (float(vals[worst]), float(got[worst]), float(ref[worst]))


# ----------------------------------------------------------------------------------------------------------------------
# the tower's linear layers on the GEMM kernel: out [M][N] = x [M][K] W^T + b (+ residual), rows after M untouched
# ----------------------------------------------------------------------------------------------------------------------
def _ulp16(ref):
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


@pytest.mark.parametrize("N,K,res", [(2304, 768, False), (768, 768, True), (3072, 768, False), (768, 3072, True),
                                     (3072, 1024, False), (1024, 1024, True), (4096, 1024, False), (1024, 4096, True)])
@pytest.mark.parametrize("M", [77, 154, 231, 616])
def test_clip_linear_shapes(M, N, K, res):
    """the tower's GEMM call (M = B x 77 token rows, one row lattice): the tower's next arena buffer follows each output
    directly, so the rows after M must come back unchanged."""
    n = _n()
    g = _gen(M + N + K)
    x = torch.randn(M, K, generator=g).half().cuda()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).half().cuda()
    bias = (torch.randn(N, generator=g) * 0.5).float().cuda()
    resid = (torch.randn(M, N, generator=g) * 2).half().cuda() if res else None
    before = [t.clone() for t in (x, w, bias, resid) if t is not None]
    wp = n.pack_weight(w)
    extra = 64
    buf = torch.full(((M + extra) * N,), SENT, dtype=torch.float16, device="cuda")
    buf[:M * N] = float("nan")
    d = n.GemmDesc()
    d.A, d.C, d.W, d.H, d.B, d.sW = x.data_ptr(), K, M, 1, 1, K
    d.Wt, d.N, d.bias = wp.data_ptr(), N, bias.data_ptr()
    if res:
        d.resid, d.ldr = resid.data_ptr(), N
    d.out, d.ldc, d.alpha = buf.data_ptr(), N, 1.0
    n.gemm(d)
    torch.cuda.synchronize()
    assert _tail_ok(buf, M * N)
    assert all(torch.equal(a, b) for a, b in zip(before, [t for t in (x, w, bias, resid) if t is not None]))
    out = buf[:M * N].view(M, N).double()
    xd, wd = x.double(), w.double()
    ref = xd @ wd.T + bias.double()
    mag = xd.abs() @ wd.abs().T + bias.double().abs()
    if res:
        ref, mag = ref + resid.double(), mag + resid.double().abs()
    # one fp16 ulp of the exact value (the one rounding) plus the fp32 accumulation where the sum cancels
    tol = _ulp16(ref) + 2.0 ** -18 * mag
    assert bool(torch.isfinite(out).all())
    assert bool(((out - ref).abs() <= tol).all()), float(((out - ref).abs() - tol).max())
