"""CPU: the LPIPS oracle (fp64 restatement on torchvision's AlexNet features), the weight loading / validation, and the packed
weight layout the kernels read."""
import pytest
import torch
import torch.nn.functional as F

from gaussianavatar_b200 import lpips as gl
from oracle import lpips_oracle as lo


def _oracle(sd=None, seed=0):
    return lo.LpipsOracle(sd if sd is not None else lo.random_state_dict(seed)).double()


@pytest.mark.parametrize("H,W", [(1024, 1024), (512, 384), (31, 31), (31, 40)])
def test_oracle_map_shapes(H, W):
    expect = lo.map_shapes(H, W)
    if (H, W) == (1024, 1024):
        assert expect == [(255, 255), (127, 127), (63, 63), (63, 63), (63, 63)]
    net = lo.LpipsOracle(lo.random_state_dict(0))
    with torch.no_grad():
        maps = net.maps(torch.rand(1, 3, H, W) * 2 - 1)
    assert [tuple(m.shape[-2:]) for m in maps] == expect
    assert [m.shape[1] for m in maps] == list(lo.CHANNELS)


@pytest.mark.parametrize("H,W", [(30, 40), (40, 30)])
def test_oracle_rejects_images_below_31(H, W):
    with pytest.raises(RuntimeError):
        lo.LpipsOracle(lo.random_state_dict(0))(torch.zeros(1, 3, H, W), torch.zeros(1, 3, H, W))


def test_oracle_gradient_matches_finite_differences():
    net = _oracle(seed=1)
    g = torch.Generator().manual_seed(2)
    x0 = (torch.rand(2, 3, 37, 33, generator=g, dtype=torch.float64) * 2 - 1).requires_grad_(True)
    x1 = torch.rand(2, 3, 37, 33, generator=g, dtype=torch.float64) * 2 - 1
    out = net(x0, x1)
    assert out.shape == (2, 1, 1, 1)
    (grad,) = torch.autograd.grad(out.sum(), x0)
    h = 1e-6
    for _ in range(3):
        v = torch.randn(x0.shape, generator=g, dtype=torch.float64)
        with torch.no_grad():
            fd = (net(x0 + h * v, x1).sum() - net(x0 - h * v, x1).sum()) / (2 * h)
        assert abs(float(fd) - float((grad * v).sum())) <= 1e-6 * max(1.0, abs(float(fd)))


def zero_feature_state_dict(seed=3):
    """conv1 with positive weights and a negative bias: a dark region of the input gives all-zero relu1 vectors, a bright one does
    not."""
    sd = lo.random_state_dict(seed)
    sd["net.slice1.0.weight"] = sd["net.slice1.0.weight"].abs()
    sd["net.slice1.0.bias"] = torch.full((64,), -0.05)
    return sd


def dark_patch_pair(B=1, H=48, W=48, seed=4):
    g = torch.Generator().manual_seed(seed)
    x0 = torch.rand(B, 3, H, W, generator=g, dtype=torch.float64) * 2 - 1
    x0[:, :, 8:40, 8:40] = -1.0                       # relu1 is all zero over this patch's interior
    x1 = torch.rand(B, 3, H, W, generator=g, dtype=torch.float64) * 0.5 + 0.5
    return x0, x1


def test_oracle_zero_feature_vector_rule():
    net = _oracle(zero_feature_state_dict())
    x0, x1 = dark_patch_pair()
    x0.requires_grad_(True)
    out = net(x0, x1)
    (grad,) = torch.autograd.grad(out.sum(), x0)
    assert torch.isfinite(grad).all()
    with torch.no_grad():
        r0, r1 = net.maps(x0)[0], net.maps(x1)[0]
    zero = (r0 == 0).all(dim=1)[0]                   # relu1 pixels whose feature vector is all zero
    assert zero[4:6, 4:6].all()
    # such a pixel contributes sum_c w_c fhat1_c^2 to the value ...
    f1 = r1 / (r1.pow(2).sum(1, keepdim=True).sqrt() + lo.EPS)
    d = (f1 ** 2 * net.lin0).sum(1)[0]
    f0 = r0 / (r0.pow(2).sum(1, keepdim=True).sqrt() + lo.EPS)
    d_all = ((f0 - f1) ** 2 * net.lin0).sum(1)[0]
    assert torch.allclose(d_all[zero], d[zero], rtol=0, atol=0)
    # ... and nothing to the gradient: input pixels that only reach all-zero relu1 vectors get exactly zero
    assert (grad[0, :, 18:30, 18:30] == 0).all()


def test_load_alex_weights_from_both_files(tmp_path):
    sd = lo.random_state_dict(5)
    lin = {lo.lin_key(k): sd[lo.lin_key(k)].clone() for k in range(5)}
    alex = {}
    for wk, bk, i in lo.conv_keys():
        alex[f"features.{i}.weight"] = sd[wk].clone()
        alex[f"features.{i}.bias"] = sd[bk].clone()
    alex["classifier.1.weight"] = torch.zeros(4, 4)                       # the classifier is there and ignored
    torch.save(lin, tmp_path / "alex.pth")
    torch.save(alex, tmp_path / "alexnet-owt.pth")
    got = gl.load_alex_weights(str(tmp_path / "alex.pth"), str(tmp_path / "alexnet-owt.pth"))
    assert set(got) == set(sd)
    for k in sd:
        assert torch.equal(got[k], sd[k]), k

    bad = dict(alex); del bad["features.6.bias"]
    torch.save(bad, tmp_path / "missing.pth")
    with pytest.raises(KeyError, match="features.6.bias"):
        gl.load_alex_weights(str(tmp_path / "alex.pth"), str(tmp_path / "missing.pth"))
    bad_lin = dict(lin); bad_lin["lin3.model.1.weight"] = torch.zeros(1, 255, 1, 1)
    torch.save(bad_lin, tmp_path / "badlin.pth")
    with pytest.raises(ValueError, match="lin3.model.1.weight"):
        gl.load_alex_weights(str(tmp_path / "badlin.pth"), str(tmp_path / "alexnet-owt.pth"))


def test_state_dict_validation():
    sd = lo.random_state_dict(6)
    full = dict(sd)
    for k in range(5):
        full[f"lins.{k}.model.1.weight"] = sd[lo.lin_key(k)].clone()
    full["scaling_layer.shift"] = torch.tensor(lo.SHIFT).reshape(1, 3, 1, 1)
    full["scaling_layer.scale"] = torch.tensor(lo.SCALE).reshape(1, 3, 1, 1)
    assert set(gl.validate_state_dict(full)) == set(sd)
    for key, val, err in [("lins.2.model.1.weight", sd["lin2.model.1.weight"] + 1, ValueError),
                          ("scaling_layer.scale", torch.ones(1, 3, 1, 1), ValueError),
                          ("net.slice1.0.weight", torch.zeros(64, 3, 11, 10), ValueError),
                          ("something.else", torch.zeros(1), KeyError)]:
        bad = dict(full); bad[key] = val
        with pytest.raises(err, match=key.replace(".", r"\.")):
            gl.validate_state_dict(bad)
    missing = dict(sd); del missing["net.slice4.8.weight"]
    with pytest.raises(KeyError, match=r"net\.slice4\.8\.weight"):
        gl.validate_state_dict(missing)


def _cols(x, k, stride, pad):
    """im2col with K ordered tap-major, channel-minor (the kernels' k = tap * C_in + ci)."""
    B, C = x.shape[:2]
    u = F.unfold(x, k, padding=pad, stride=stride)                   # [B, C*k*k, L], channel-major
    return u.view(B, C, k * k, -1).permute(0, 2, 1, 3).reshape(B, k * k * C, -1)


def test_packed_weight_layout():
    """The forward and data-gradient GEMMs over the packed buffer reproduce conv2d and its input gradient."""
    sd = lo.random_state_dict(7)
    flat = gl.pack_weights(sd, "cpu").double()
    off = 0
    g = torch.Generator().manual_seed(8)
    fwd = []
    for k in range(5):
        cin, cout, ks = lo.IN_CHANNELS[k], lo.CHANNELS[k], lo.KERNELS[k]
        K = 384 if k == 0 else ks * ks * cin
        fwd.append((flat[off:off + cout * K].view(cout, K), flat[off + cout * K:off + cout * K + cout]))
        off += cout * K + cout
    dgrad = {}
    for k in range(1, 5):
        cin, cout, ks = lo.IN_CHANNELS[k], lo.CHANNELS[k], lo.KERNELS[k]
        dgrad[k] = flat[off:off + cin * ks * ks * cout].view(cin, ks * ks * cout)
        off += cin * ks * ks * cout
    for k in range(5):
        assert torch.equal(flat[off:off + lo.CHANNELS[k]], sd[lo.lin_key(k)].double().reshape(-1))
        off += lo.CHANNELS[k]
    assert off == flat.numel()
    for k, (wk, bk, _) in enumerate(lo.conv_keys()):
        w, b = sd[wk].double(), sd[bk].double()
        cin, ks = lo.IN_CHANNELS[k], lo.KERNELS[k]
        stride, pad = (4, 2) if k == 0 else (1, ks // 2)
        x = torch.randn(2, cin, 23, 19, generator=g, dtype=torch.float64)
        ref = F.conv2d(x, w, b, stride=stride, padding=pad)
        Wp, bp = fwd[k]
        cols = _cols(x, ks, stride, pad)
        got = (Wp[:, :cols.shape[1]] @ cols + bp[:, None]).view(ref.shape)
        assert torch.allclose(got, ref, atol=1e-10)
        if k == 0:
            assert (Wp[:, 363:] == 0).all()
            continue
        dy = torch.randn(ref.shape, generator=g, dtype=torch.float64)
        ref_dx = torch.nn.grad.conv2d_input(x.shape, w, dy, stride=1, padding=pad)
        got_dx = (dgrad[k] @ _cols(dy, ks, 1, pad)).view(ref_dx.shape)
        assert torch.allclose(got_dx, ref_dx, atol=1e-10)


def test_oracle_matches_lpips_package():
    lpips = pytest.importorskip("lpips")
    ref = lpips.LPIPS(pretrained=False, pnet_rand=True, net="alex", verbose=False).eval()
    sd = lo.random_state_dict(9)
    ref.load_state_dict({**ref.state_dict(), **sd, **{f"lins.{k}.model.1.weight": sd[lo.lin_key(k)] for k in range(5)}})
    net = lo.LpipsOracle(sd)
    g = torch.Generator().manual_seed(10)
    x0, x1 = (torch.rand(2, 3, 64, 48, generator=g) * 2 - 1 for _ in range(2))
    with torch.no_grad():
        assert torch.allclose(net(x0, x1), ref(x0, x1), rtol=1e-5, atol=1e-7)
