"""Fine-tuning without a GPU: the per-unit backward plan of partially frozen networks (which units run a weight gradient,
where the backward stops, which units record), BatchNorm modules recognisable as nn.BatchNorm2d with the state_dict unchanged,
and the argument checks of the masked Adam entry point."""
import pytest
import torch
import torch.nn as nn


def _nets():
    import models
    from scsfm import nets as N
    return models, N


def _convs(net, N):
    return [(n, m) for n, m in net.named_modules() if isinstance(m, N.ConvParams)]


def _plan(net, dimg):
    from scsfm import nets as N
    return N.BackwardPlan(net, dimg)


@pytest.mark.parametrize("layers", [18, 50])
def test_batchnorm_modules_are_batchnorm2d_with_the_same_state_dict(layers):
    import models
    from oracle import nets as ON
    torch.manual_seed(0)
    mine = models.DispResNet(layers, False)
    ref = ON.DispResNet(layers)
    assert list(mine.state_dict()) == list(ref.state_dict())
    bns = [m for m in mine.modules() if isinstance(m, nn.BatchNorm2d)]
    assert len(bns) == sum(isinstance(m, nn.BatchNorm2d) for m in ref.modules()) > 0
    for bn in bns:
        assert torch.equal(bn.weight, torch.ones_like(bn.weight)) and torch.equal(bn.bias, torch.zeros_like(bn.bias))
        assert torch.equal(bn.running_mean, torch.zeros_like(bn.running_mean))
        assert torch.equal(bn.running_var, torch.ones_like(bn.running_var))
        assert bn.num_batches_tracked.dtype == torch.long and int(bn.num_batches_tracked) == 0
        assert (bn.momentum, bn.eps) == (0.1, 1e-5)
    # the reference's tensors load strictly, values and the BatchNorm buffers included
    sd = {k: v + 0.25 if v.is_floating_point() else v + 3 for k, v in ref.state_dict().items()}
    mine.load_state_dict(sd)
    for k, v in mine.state_dict().items():
        assert torch.equal(v, sd[k]), k
    # per-module mode, as for nn.BatchNorm2d
    mine.train()
    mine.encoder.eval()
    assert not any(bn.training for bn in bns) and mine.training and mine.decoder.training


def test_batchnorm_module_is_not_callable_and_refuses_other_hyper_parameters():
    _, N = _nets()
    bn = N.BNParams(8)
    bn.check_supported()
    with pytest.raises(RuntimeError, match="kernels"):
        bn(torch.zeros(1, 8, 2, 2))
    for attr, value in (("momentum", 0.01), ("momentum", None), ("eps", 1e-3)):
        b = N.BNParams(8)
        setattr(b, attr, value)
        with pytest.raises(ValueError, match="momentum"):
            b.check_supported()


def test_all_trainable_plan_runs_every_unit():
    models, N = _nets()
    for net, n_img in ((models.DispResNet(18, False), 1), (models.PoseResNet(18, False), 2)):
        for dimg in ((False,) * n_img, (True,) * n_img):
            p = _plan(net, dimg)
            assert p.any and all(p.feats)
            for name, conv in _convs(net, N):
                assert p.runs[id(conv)] and p.wgrad(conv), name
            # the data gradient into the stem runs only for images that need one
            assert p.dgrad[id(net.encoder.encoder.conv1)] == any(dimg)


def test_disp_encoder_frozen_backward_stops_at_the_decoder():
    models, N = _nets()
    net = models.DispResNet(18, False)
    net.encoder.requires_grad_(False)
    net.encoder.eval()
    p = _plan(net, (False,))
    assert p.any and not any(p.feats)              # no d_skip / d_feats, no encoder backward, no encoder record
    for name, conv in _convs(net, N):
        assert p.runs[id(conv)] == name.startswith("decoder"), name
        assert p.wgrad(conv) == name.startswith("decoder"), name
    # the first decoder convolution consumes the encoder's output: weight gradient, no data gradient
    assert not p.dgrad[id(net.decoder.up(4, 0))] and p.dgrad[id(net.decoder.up(4, 1))]
    # with the image needing a gradient: every data gradient returns, no encoder weight gradient
    p = _plan(net, (True,))
    assert all(p.feats)
    for name, conv in _convs(net, N):
        assert p.runs[id(conv)] and p.wgrad(conv) == name.startswith("decoder"), name
    for bn in net.encoder.modules():
        if isinstance(bn, nn.BatchNorm2d):
            assert not p.trains(bn.weight) and not p.trains(bn.bias)


def test_stem_and_layer1_frozen_backward_stops_in_layer2():
    models, N = _nets()
    for net, n_img in ((models.DispResNet(18, False), 1), (models.PoseResNet(50, False), 2)):
        t = net.encoder.encoder
        for m in (t.conv1, t.bn1, t.layer1):
            m.requires_grad_(False)
        p = _plan(net, (False,) * n_img)
        assert p.feats == [False, False, True, True, True]
        assert not p.runs[id(t.conv1)]
        for blk in t.layer1:
            main, ds = blk.units()
            assert not any(p.runs[id(u[0])] for u in main)
            assert ds is None or not p.runs[id(ds[0])]
        first = t.layer2[0]
        main, ds = first.units()
        # layer2's first block runs every unit and its weight gradients, but no data gradient into layer1
        assert all(p.runs[id(u[0])] and p.wgrad(u[0]) for u in main + [ds])
        assert not p.dgrad[id(main[0][0])] and not p.dgrad[id(ds[0])]
        assert all(p.dgrad[id(u[0])] for u in main[1:])


def test_decoder_frozen_runs_everything_but_decoder_weight_gradients():
    models, N = _nets()
    for net, n_img in ((models.DispResNet(18, False), 1), (models.PoseResNet(18, False), 2)):
        net.decoder.requires_grad_(False)
        p = _plan(net, (False,) * n_img)
        assert all(p.feats)
        for name, conv in _convs(net, N):
            assert p.runs[id(conv)] and p.wgrad(conv) == name.startswith("encoder"), name


def test_whole_network_frozen_has_no_backward_unless_an_image_needs_one():
    models, N = _nets()
    net = models.PoseResNet(18, False)
    net.requires_grad_(False)
    p = _plan(net, (False, False))
    assert not p.any and not p.train
    p = _plan(net, (False, True))
    assert p.any and all(p.feats) and not any(p.wgrad(c) for _, c in _convs(net, N))


def test_batchnorm_affine_frozen_and_weight_only_frozen_units():
    models, N = _nets()
    net = models.DispResNet(18, False)
    for m in net.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.requires_grad_(False)
    p = _plan(net, (False,))
    assert all(p.feats) and all(p.wgrad(c) for _, c in _convs(net, N))
    assert not p.trains(net.encoder.encoder.bn1.weight)
    # a decoder convolution whose weight is frozen while its bias trains: the unit still runs its weight-gradient kernel
    net = models.DispResNet(18, False)
    c = net.decoder.up(2, 1)
    c.weight.requires_grad_(False)
    p = _plan(net, (False,))
    assert p.wgrad(c) and not p.trains(c.weight) and p.trains(c.bias)
    # the pose head is a chain: only its last convolution trains -> the backward is that one weight gradient
    net = models.PoseResNet(18, False)
    net.requires_grad_(False)
    net.decoder.net[3].requires_grad_(True)
    p = _plan(net, (False, False))
    assert [p.runs[id(c)] for c in net.decoder.net] == [False, False, False, True]
    assert not p.dgrad[id(net.decoder.net[3])] and not any(p.feats)


def test_no_gradient_without_autograd():
    models, N = _nets()
    net = models.DispResNet(18, False)
    with torch.no_grad():
        p = _plan(net, (False,))
    assert not p.any and not p.train


def test_masked_adam_entry_point_rejects_bad_arguments_without_a_gpu():
    from scsfm import lib
    from scsfm import nnops as O
    L = O._lib()
    assert L.scsfm_adam_step_masked(None, None, None, None, 64, None, 1e-4, 0.9, 0.999, 1e-8, 0.0, 1, None, None, 0, None) == -1
    assert b"adam_step_masked" in lib.load().scsfm_last_error()
    # every pointer present but the mask, then a bad step count, then a bad mirror operand kind
    p = 16          # a non-null address: each call fails its checks before anything is launched
    assert L.scsfm_adam_step_masked(p, p, p, p, 64, None, 1e-4, 0.9, 0.999, 1e-8, 0.0, 1, None, None, 0, None) == -1
    assert L.scsfm_adam_step_masked(p, p, p, p, 64, p, 1e-4, 0.9, 0.999, 1e-8, 0.0, 0, None, None, 0, None) == -1
    assert L.scsfm_adam_step_masked(p, p, p, p, 64, p, 1e-4, 0.9, 0.999, 1e-8, 0.0, 1, None, None, 1, None) == -1
    assert b"mirror" in lib.load().scsfm_last_error()
    assert L.scsfm_adam_step_masked(p, p, p, p, 0, p, 1e-4, 0.9, 0.999, 1e-8, 0.0, 1, None, None, 0, None) == -1
    x = torch.zeros(130)
    with pytest.raises(ValueError, match="chunk_mask"):
        O.adam_step_masked(x, x, x, x, torch.ones(2, dtype=torch.uint8), 1e-4, 0.9, 0.999, 1e-8, 0.0, 1)
    with pytest.raises(ValueError, match="chunk_mask"):
        O.adam_step_masked(x, x, x, x, torch.ones(3, dtype=torch.int32), 1e-4, 0.9, 0.999, 1e-8, 0.0, 1)


def test_chunk_mask_covers_each_trainable_tensor_and_its_padding():
    from scsfm import nnops as O
    m = O.chunk_mask([10, 64, 65, 1], [True, False, True, False], "cpu")
    assert m.tolist() == [1, 0, 1, 1, 0]
