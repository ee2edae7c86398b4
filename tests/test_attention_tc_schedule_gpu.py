"""GPU: the wgmma flash attention's pipelined schedule (S(j+1) issued before the softmax of tile j, the two consumer warpgroups
taking turns on the tensor cores, the 64-wide grid's rel-pos bias held in registers) vs fp64 softmax attention.  Long key loops
wrap the 3-stage ring and the turn barriers many times; T = 256 runs the shortest loop; a +-30 rel-pos range moves the row max
between tiles, so the online-softmax correction is exercised."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops(cuda):
    from hipie_b200 import ops as o
    o.set_precision(3)
    return o


def _attn_ref(q, k, v, scale, rel_h, rel_w, kh, kw):
    # q, k, v: (B, H, T, hd) double
    s = (q * scale) @ k.transpose(-1, -2)
    B, H, Tq, _ = q.shape
    s = (s.view(B, H, Tq, kh, kw) + rel_h.double()[..., :, None] + rel_w.double()[..., None, :]).view(B, H, Tq, kh * kw)
    return torch.softmax(s, -1) @ v


# (grid rows, grid columns, batch): 64-wide global grids (4096 tokens, and the 256-token minimum), the 80-wide grid of 1280-pixel
# inputs, the 14 x 14 windows
SHAPES = {"g4096": (64, 64, 1), "g256": (4, 64, 2), "w80": (16, 80, 1), "win": (14, 14, 5)}


def _inputs(cuda, shape, rel_range, seed):
    gh, gw, B = SHAPES[shape]
    H, hd = 2, 80
    T, E = gh * gw, H * hd
    g = torch.Generator(device="cuda").manual_seed(seed)
    qk = torch.randn(B * T, 2 * E, device=cuda, generator=g)
    v = torch.randn(B * T, E, device=cuda, generator=g)
    rel_h = (torch.rand(B, H, T, gh, device=cuda, generator=g) * 2 - 1) * rel_range
    rel_w = (torch.rand(B, H, T, gw, device=cuda, generator=g) * 2 - 1) * rel_range
    if shape == "win":          # V^T holds every window at a 200-column pitch, pad columns zero
        vt = torch.zeros(E, B, 200, device=cuda)
        vt[:, :, :T] = v.t().reshape(E, B, T)
        vt = vt.view(E, B * 200)
    else:
        vt = v.t().contiguous()
    return B, H, hd, gh, gw, T, E, qk, vt, rel_h, rel_w


def _v_of(vt, B, T, E, win):
    vt = vt.float()
    return (vt.view(E, B, 200)[:, :, :T].reshape(E, B * T) if win else vt).t()


@pytest.mark.parametrize("rel_range", [1.0, 30.0])
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("mode", ["f16", "p3"])
def test_attention_tc_schedule(ops, cuda, mode, shape, rel_range):
    B, H, hd, gh, gw, T, E, qk, vt, rel_h, rel_w = _inputs(cuda, shape, rel_range, 7 + SHAPES[shape][0] + int(rel_range))
    sh = lambda x: x.reshape(B, T, H, hd).permute(0, 2, 1, 3).double()
    args = (B, H, T, hd, T * 2 * E, 2 * E, T * 2 * E, 2 * E, hd ** -0.5)
    rel = dict(rel_h=rel_h, rel_w=rel_w, kh=gh, kw=gw)
    if mode == "f16":
        qk16, vt16 = qk.half(), vt.half()
        q, k, vs = ops.BF2(qk16[:, :E], None), ops.BF2(qk16[:, E:], None), ops.BF2(vt16, None)
        o, _ = ops.attention_tc(q, k, vs, *args, want_f32=True, want_split=False, f16=True, **rel)
        ref = _attn_ref(sh(qk16[:, :E].float()), sh(qk16[:, E:].float()), sh(_v_of(vt16, B, T, E, shape == "win")), hd ** -0.5,
                        rel_h, rel_w, gh, gw)
        tol = 2e-3                 # P is rounded to fp16 before the PV pass
        # the fp16 + e4m3 output planes of the same call are the split of the fp32 output
        _, s = ops.attention_tc(q, k, vs, *args, out_e4m3=True, f16=True, **rel)
        planes = ops.split_f16_e4m3(o.view(B * T, E))
        assert torch.equal(s.hi.view(B * T, E), planes.hi) and torch.equal(s.lo.view(B * T, 2 * E), planes.lo)
    else:
        S, Vs = ops.split(qk), ops.split(vt)
        q, k = ops.BF2(S.hi[:, :E], S.lo[:, :E]), ops.BF2(S.hi[:, E:], S.lo[:, E:])
        o, _ = ops.attention_tc(q, k, Vs, *args, want_f32=True, want_split=False, prec=3, **rel)
        ref = _attn_ref(sh(qk[:, :E]), sh(qk[:, E:]), sh(_v_of(vt, B, T, E, shape == "win")), hd ** -0.5, rel_h, rel_w, gh, gw)
        tol = 3e-5
    err = (o.double() - ref.permute(0, 2, 1, 3).reshape(B, T, E)).abs().max().item()
    assert err < tol, err
