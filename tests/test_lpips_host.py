"""CPU: weight loading and argument handling of vtoonify_b200.lpips.PerceptualLoss (no kernels run)."""
import pytest
import torch

from tests import oracle_lpips as O
from vtoonify_b200.lpips import VGG_CONVS, PerceptualLoss, PNetLin, default_model_path, vgg_state_dict
from vtoonify_b200.weights import det_state_dict


def _vgg16_file(path, seed=0):
    """a torchvision-vgg16-format checkpoint: `features.{i}` for every conv, plus the classifier entries the loader ignores"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i, (_, cin, cout) in VGG_CONVS.items():
        sd[f"features.{i}.weight"] = torch.randn(cout, cin, 3, 3, generator=g)
        sd[f"features.{i}.bias"] = torch.randn(cout, generator=g)
    sd["classifier.0.weight"] = torch.randn(4, 4, generator=g)
    torch.save(sd, path)
    return sd


def _lin_file(path, seed=1):
    g = torch.Generator().manual_seed(seed)
    sd = {f"lin{k}.model.1.weight": torch.rand(1, c, 1, 1, generator=g) for k, c in enumerate(O.CHANNELS)}
    torch.save(sd, path)
    return sd


def test_torchvision_key_mapping():
    src = {f"features.{i}.{p}": torch.tensor(float(i)) for i in VGG_CONVS for p in ("weight", "bias")}
    out = vgg_state_dict(src)
    assert len(out) == 26
    assert out["net.slice1.0.weight"] == 0 and out["net.slice2.7.bias"] == 7 and out["net.slice3.14.weight"] == 14
    assert out["net.slice4.17.bias"] == 17 and out["net.slice5.28.weight"] == 28
    del src["features.19.weight"]
    with pytest.raises(KeyError, match="features.19.weight"):
        vgg_state_dict(src)


def test_loads_local_weight_files(tmp_path):
    vgg = _vgg16_file(tmp_path / "vgg16.pth")
    lin = _lin_file(tmp_path / "vgg.pth")
    p = PerceptualLoss(model="net-lin", net="vgg", use_gpu=False, vgg_path=str(tmp_path / "vgg16.pth"), model_path=str(tmp_path / "vgg.pth"))
    sd = p.model.net.state_dict()
    assert len(sd) == 33
    for i, (s, _, _) in VGG_CONVS.items():
        assert torch.equal(sd[f"net.slice{s}.{i}.weight"], vgg[f"features.{i}.weight"])
        assert torch.equal(sd[f"net.slice{s}.{i}.bias"], vgg[f"features.{i}.bias"])
    for k, v in lin.items():
        assert torch.equal(sd[k], v)
    assert torch.equal(sd["scaling_layer.scale"].flatten(), torch.tensor([.458, .448, .450]))
    assert not p.model.net.training
    assert all(not q.requires_grad for q in p.model.net.net.parameters())
    assert p.model.name() == "net-lin [vgg]"


def test_missing_files_raise(tmp_path, monkeypatch):
    _lin_file(tmp_path / "vgg.pth")
    with pytest.raises(FileNotFoundError, match="nope.pth"):
        PerceptualLoss(net="vgg", use_gpu=False, vgg_path=str(tmp_path / "nope.pth"), model_path=str(tmp_path / "vgg.pth"))
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    with pytest.raises(FileNotFoundError, match="vgg16-397923af.pth"):
        PerceptualLoss(net="vgg", use_gpu=False, model_path=str(tmp_path / "vgg.pth"))
    with pytest.raises(FileNotFoundError, match="missing_lin.pth"):
        PerceptualLoss(net="vgg", use_gpu=False, pnet_rand=True, model_path=str(tmp_path / "missing_lin.pth"))


def test_default_lin_path_is_next_to_the_reference_package(tmp_path, monkeypatch):
    pkg = tmp_path / "model" / "stylegan" / "lpips"
    pkg.mkdir(parents=True)
    for d in (tmp_path / "model", tmp_path / "model" / "stylegan"):
        (d / "__init__.py").write_text("")
    (pkg / "__init__.py").write_text("raise RuntimeError('the lpips package must not be executed')\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    for m in [m for m in list(__import__("sys").modules) if m == "model" or m.startswith("model.")]:
        monkeypatch.delitem(__import__("sys").modules, m)
    assert default_model_path("vgg") == str(pkg / "weights" / "v0.1" / "vgg.pth")
    with pytest.raises(FileNotFoundError, match="weights/v0.1/vgg.pth"):
        PerceptualLoss(net="vgg", use_gpu=False, pnet_rand=True)


@pytest.mark.parametrize("kw,name", [({"net": "alex"}, "net"), ({"net": "squeeze"}, "net"), ({"model": "net", "net": "vgg"}, "model"),
                                     ({"model": "L2", "net": "vgg"}, "model"), ({"net": "vgg", "spatial": True}, "spatial")])
def test_unsupported_arguments_raise(kw, name):
    with pytest.raises(NotImplementedError, match=name):
        PerceptualLoss(use_gpu=False, pnet_rand=True, **kw)


def test_default_net_is_the_reference_default():
    with pytest.raises(NotImplementedError, match="'alex'"):
        PerceptualLoss(use_gpu=False)


def test_strict_load_of_the_oracle_state_dict():
    sd = det_state_dict(PNetLin(pnet_rand=True), seed=3)
    net = PNetLin(pnet_rand=True)
    net.load_state_dict(sd, strict=True)
    assert all(torch.equal(net.state_dict()[k], v) for k, v in sd.items())


def test_pnet_rand_is_deterministic():
    a, b = PNetLin(pnet_rand=True).state_dict(), PNetLin(pnet_rand=True).state_dict()
    assert all(torch.equal(a[k], b[k]) for k in a if k.startswith("net."))


def test_grad_mode_rejects_trainable_parameters():
    net = PNetLin(pnet_rand=True)
    x = torch.zeros(1, 3, 16, 16)
    with torch.enable_grad(), pytest.raises(NotImplementedError, match="lin0.model.1.weight"):
        net(x, x)
