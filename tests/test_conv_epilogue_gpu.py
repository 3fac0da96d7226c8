"""The store phase of the persistent fprop / dgrad kernel (conv_gemm_pp): whole 16-byte bf16 chunks under beta != 0 go
through a batched path that loads a batch's old values before its stores; beta == 0, partial chunks and unaligned pitches
store one chunk at a time.  Every case checks, bit for bit, that the beta result is the kernel's own beta = 0 result
accumulated as the kernel defines it (fp32 value + beta * old, rounded to bf16 once), that nothing outside the output's
rows and channel slice is written, and that a second run gives the same bits."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from seg_b200 import ops
    from seg_b200.lib import IMPL_TC

DEV = "cuda"
SENTINEL = -777.0  # exactly representable in bf16

# (kind, N, H, C, K, ksize, stride, pad, beta, slice): fprop writes K channels, dgrad writes C; `slice` = (offset, width) of
# the channel slice written inside a wider buffer, or None
CASES = [
    ("dgrad", 2, 33, 256, 64, 1, 1, 0, 1.0, None),       # 1 k-block per tile, 17 row tiles (the last one 2 rows)
    ("dgrad", 2, 33, 256, 1024, 1, 1, 0, 1.0, None),     # 16 k-blocks per tile
    ("dgrad", 2, 33, 200, 256, 1, 1, 0, 1.0, None),      # column tail: the second 128-wide tile has 72 columns
    ("dgrad", 2, 33, 200, 256, 1, 1, 0, 0.0, None),
    ("dgrad", 2, 33, 256, 256, 1, 1, 0, 0.5, (64, 256)),  # concat slice: channels 64..319 of 384
    ("dgrad", 2, 33, 128, 128, 3, 2, 1, 1.0, None),      # stride 2: four parity classes on strided sub-grids
    ("dgrad", 2, 33, 128, 128, 3, 2, 1, 1.0, (8, 128)),  # ... into a channel slice
    ("fprop", 2, 33, 256, 1024, 1, 1, 0, 1.0, None),     # 4 k-blocks, 8 column tiles
    ("fprop", 2, 33, 64, 64, 3, 1, 1, 0.5, (16, 64)),    # 64-wide tiles into a slice
    ("fprop", 2, 33, 64, 19, 1, 1, 0, 1.0, None),        # 19 channels: pitch of 38 bytes, partial chunks
]


def case_id(c):
    kind, n, h, cin, k, ks, s, pad, beta, sl = c
    return f"{kind}-{n}x{h}-{cin}to{k}-k{ks}s{s}-beta{beta:g}" + (f"-slice{sl[0]}" if sl else "")


def run(case, old):
    """One launch into a copy of the guarded buffer `old`; returns the whole buffer."""
    kind, n, h, cin, k, ks, s, pad, beta, sl = case
    g = torch.Generator(device=DEV).manual_seed(7)
    p = (h + 2 * pad - ks) // s + 1
    w = torch.randn(k, cin, ks, ks, device=DEV, generator=g) / (cin * ks * ks) ** 0.5
    wp = ops.pack_weight(w)
    buf = old.clone()
    out = buf if sl is None else buf[..., sl[0]:sl[0] + sl[1]]
    if kind == "dgrad":
        dy = torch.randn(n, p, p, k, device=DEV, generator=g).to(torch.bfloat16)
        ops.conv2d_dgrad(dy, wp, (n, h, h, cin), ks, ks, s, pad, 1, out=out, beta=beta, impl=IMPL_TC)
    else:
        x = torch.randn(n, h, h, cin, device=DEV, generator=g).to(torch.bfloat16)
        ops.conv2d_fwd(x, wp, k, ks, ks, s, pad, 1, out=out, beta=beta, impl=IMPL_TC)
    torch.cuda.synchronize()
    return buf


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_store_phase(case):
    kind, n, h, cin, k, ks, s, pad, beta, sl = case
    p = (h + 2 * pad - ks) // s + 1
    hw, ch = (h, cin) if kind == "dgrad" else (p, k)
    width = ch if sl is None else sl[0] + sl[1] + 64
    g = torch.Generator(device=DEV).manual_seed(11)
    old = torch.randn(n, hw, hw, width, device=DEV, generator=g).to(torch.bfloat16)
    lo, hi = (0, ch) if sl is None else (sl[0], sl[0] + sl[1])
    if sl is not None:
        old[..., :lo] = SENTINEL
        old[..., hi:] = SENTINEL
    y = run(case, old)
    assert torch.equal(y.view(torch.int16), run(case, old).view(torch.int16)), "two runs differ"
    if sl is not None:
        assert torch.equal(y[..., :lo], old[..., :lo]) and torch.equal(y[..., hi:], old[..., hi:]), "wrote outside the slice"
    # the beta = 0 result of the same kernel, into a fresh buffer
    y0 = run((kind, n, h, cin, k, ks, s, pad, 0.0, sl), torch.full_like(old, SENTINEL))
    got, base, prev = y[..., lo:hi], y0[..., lo:hi], old[..., lo:hi]
    # bf16 + beta * bf16 (beta in {0, 0.5, 1}) is exact in float64, so its rounding to fp32 is the kernel's single fp32
    # rounding of fma(beta, old, value); then the one rounding to bf16
    want = (base.double() + beta * prev.double()).float().to(torch.bfloat16)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), \
        f"{(got.float() != want.float()).sum().item()} elements differ from value + beta * old"
