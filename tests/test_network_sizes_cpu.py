"""The image sizes DispResNet and the training step take, and the shape checks of the decoder's upsample + concatenation.

DispResNet's decoder concatenates every x2 upsampled stage with an encoder feature, so a size whose encoder planes do not
halve exactly has no valid concatenation: the reference's torch.cat raises, and this project's upsample + concat kernel would
read the skip feature at the wrong strides and past its end.  scsfm.nets.check_image_size restates the reference's rule; the
sweep below pins it to what the fp32 oracle module (the reference's layers) actually runs.  No GPU needed."""
import pytest
import torch

SIDES = range(2, 130)


def _oracle_runs(net, H, W):
    try:
        with torch.no_grad():
            return tuple(net(torch.zeros(1, 3, H, W)).shape)
    except RuntimeError:
        return None


def test_size_rule_is_the_reference_modules_rule():
    """H in 2..129 at W = 64 and W in 2..129 at H = 64: the oracle DispResNet-18 eval forward runs exactly where
    check_image_size accepts the size, and then gives a 2 ceil(H/2) x 2 ceil(W/2) disparity."""
    from oracle import nets as ON
    from scsfm.nets import check_image_size
    torch.manual_seed(0)
    net = ON.DispResNet(18).eval()
    accepted = []
    for H, W in [(h, 64) for h in SIDES] + [(64, w) for w in SIDES]:
        try:
            check_image_size(H, W)
            ok = True
        except ValueError:
            ok = False
        got = _oracle_runs(net, H, W)
        assert (got is not None) == ok, (H, W, got, ok)
        if ok:
            assert got == (1, 1, 2 * ((H + 1) // 2), 2 * ((W + 1) // 2)), (H, W, got)
            accepted.append((H, W))
    assert accepted == [(h, 64) for h in (63, 64, 95, 96, 127, 128)] + [(64, w) for w in (63, 64, 95, 96, 127, 128)]


def test_training_step_sizes():
    """A training step takes multiples of 32 from 64 up (the disparity at the image's size, and a size DispResNet takes)."""
    from scsfm.nets import check_image_size
    for n in range(2, 1300):
        try:
            check_image_size(n, 64, training_step=True)
            check_image_size(64, n, training_step=True)
            ok = True
        except ValueError:
            ok = False
        assert ok == (n % 32 == 0 and n >= 64), n
        if ok:
            check_image_size(n, n)                   # a DispResNet size too
    with pytest.raises(ValueError, match=r"255x831: .*multiples of 32.*nearest accepted sizes: 256x832, 224x832, 256x800, 224x800"):
        check_image_size(255, 831, training_step=True)


@pytest.mark.parametrize("size, nearest", [((250, 832), "255x832, 224x832"), ((256, 830), "256x831, 256x800"),
                                           ((375, 1242), "383x1247, 352x1247, 383x1216, 352x1216"), ((30, 64), "63x64"),
                                           ((62, 2), "63x63")])
def test_refusal_names_the_size_and_the_nearest_accepted_sizes(size, nearest):
    from scsfm.nets import check_image_size
    H, W = size
    with pytest.raises(ValueError) as e:
        check_image_size(H, W)
    msg = str(e.value)
    assert msg.startswith("image size %dx%d: " % (H, W)) and msg.endswith("(nearest accepted sizes: %s)" % nearest), msg


def test_disp_resnet_refuses_before_anything_else():
    """A refused size raises ValueError in forward and forward_multi, eval and train mode, before the module even asks for its
    device (a CPU module at an accepted size raises the no-CPU-fallback RuntimeError instead)."""
    import models
    from scsfm import lib
    net = models.DispResNet(18, False)
    n0 = lib.launch_count()
    for training in (False, True):
        net.train(training)
        for H, W in ((250, 832), (256, 830), (375, 1242), (30, 64)):
            x = torch.zeros(1, 3, H, W)
            with pytest.raises(ValueError, match="image size %dx%d" % (H, W)):
                net(x)
            with pytest.raises(ValueError, match="image size %dx%d" % (H, W)):
                net.forward_multi([torch.zeros(1, 3, 64, 64), x])
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            net(torch.zeros(1, 3, 255, 831))
    assert lib.launch_count() == n0 and net._pending == 0


@pytest.mark.parametrize("skip_shape", [(2, 7, 12, 12), (2, 8, 11, 12), (1, 8, 12, 12), (3, 8, 12, 12), (2, 9, 12, 12),
                                        (2, 4, 6, 12)])
def test_upcat_and_fold_refuse_a_mismatched_skip_before_any_launch(skip_shape):
    """upcat_fwd with a skip one row or one column short or long, or of another batch, and fold_upcat with the gradient of the
    matching padded concatenation, raise ValueError without a launch (the checks come first, so CPU tensors do)."""
    from scsfm import lib
    from scsfm import nnops as O
    lo = torch.zeros(2, 4, 6, 8)                     # its skip would be [2, 8, 12, C2]
    skip = torch.zeros(skip_shape)
    n0 = lib.launch_count()
    with pytest.raises(ValueError, match="upcat_fwd: skip is"):
        O.upcat_fwd(lo, skip)
    B, H, W, C2 = skip_shape
    dpad = torch.zeros(B, H + 2, W + 2, lo.shape[-1] + C2)
    for with_skip in (True, False):
        with pytest.raises(ValueError, match="fold_upcat: dpad is"):
            O.fold_upcat(dpad, lo.shape[-1], lo, O.ACT_ELU, with_skip=with_skip)
    assert lib.launch_count() == n0
