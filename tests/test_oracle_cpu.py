"""CPU tests of the oracle: hand-computable known answers for every TF1-semantics op + the golden snapshot."""
import os

import numpy as np
import torch

from oracle import tf1_ops as T
from oracle.madnet import MadNetOracle, init_params, param_shapes, mad_groups_full
from oracle.adaptation import OracleAdapter

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'madnet_64x128.npz')


def test_same_pad_table():
    # SURVEY §8c item 1: 3x3 s2 even -> (0,1); 3x3 s1 -> (1,1); 5x5 s2 -> (1,2); 7x7 s2 -> (2,3); dilated r -> (r,r)
    assert T.same_pad(8, 3, 2) == (4, 0, 1)
    assert T.same_pad(8, 3, 1) == (8, 1, 1)
    assert T.same_pad(8, 5, 2) == (4, 1, 2)
    assert T.same_pad(8, 7, 2) == (4, 2, 3)
    assert T.same_pad(32, 3, 1, 16) == (32, 16, 16)
    assert T.same_pad(7, 3, 2) == (4, 1, 1)


def test_conv_same_stride2_asymmetric():
    # single 1 at the last column must reach the last output through the pad-after column only
    x = torch.zeros(1, 4, 4, 1); x[0, 3, 3, 0] = 1.0
    w = torch.arange(9, dtype=torch.float32).view(3, 3, 1, 1)
    y = T.conv2d(x, w, torch.zeros(1), stride=2)
    # out[1,1] covers input rows/cols 2..4 (pad 0 before, 1 after): tap (1,1) hits (3,3)
    assert y.shape == (1, 2, 2, 1)
    assert float(y[0, 1, 1, 0]) == 4.0 and float(y[0, 0, 0, 0]) == 0.0


def test_conv_transpose_matches_conv_gradient():
    torch.manual_seed(0)
    x = torch.randn(1, 3, 4, 2)
    w = torch.randn(4, 4, 3, 2)        # [kh,kw,cout,cin]
    y = T.conv2d_transpose(x, w, torch.zeros(3), stride=2)
    assert y.shape == (1, 6, 8, 3)
    # definition: gradient of the SAME stride-2 conv (HWIO = [4,4,3,2]) wrt its input
    inp = torch.zeros(1, 6, 8, 3, requires_grad=True)
    z = T.conv2d(inp, w, torch.zeros(2), stride=2)
    (g,) = torch.autograd.grad(z, inp, grad_outputs=x)
    assert torch.allclose(y, g, atol=1e-5)


def test_resize_legacy_known_answer():
    x = torch.tensor([0.0, 10.0]).view(1, 1, 2, 1)
    y = T.resize_bilinear(x, 1, 4).view(-1)
    # src = dst*0.5 -> 0,0.5,1,1.5 ; hi clamps to 1
    assert torch.allclose(y, torch.tensor([0.0, 5.0, 10.0, 10.0]))
    assert T.resize_bilinear(x, 1, 2) is x


def test_crop_and_reflect():
    x = torch.arange(5, dtype=torch.float32).view(1, 1, 5, 1)
    p = T.pad_reflect_to_multiple(x.expand(1, 5, 5, 1), 8)
    assert p.shape == (1, 8, 8, 1)
    assert p[0, 1, :, 0].tolist() == [1.0, 0.0, 1.0, 2.0, 3.0, 4.0, 3.0, 2.0]   # pad 1 left, 2 right
    c = T.crop_or_pad(p, 5, 5)
    assert torch.equal(c, x.expand(1, 5, 5, 1))


def test_correlation_known_answer():
    # the B=2,H=3,W=7,C=5,d=2 case of SURVEY §4: compare with a literal loop
    rng = np.random.default_rng(0)
    a = rng.standard_normal((2, 3, 7, 5)).astype(np.float32)
    b = rng.standard_normal((2, 3, 7, 5)).astype(np.float32)
    ref = np.zeros((2, 3, 7, 5), np.float32)
    for i in range(5):
        for x in range(7):
            xs = x + i - 2
            if 0 <= xs < 7:
                ref[:, :, x, i] = (a[:, :, x] * b[:, :, xs]).mean(-1)
    out = T.correlation(torch.tensor(a), torch.tensor(b), 2).numpy()
    assert np.allclose(out, ref, atol=1e-6)
    out2 = T.correlation(torch.tensor(a), torch.tensor(b), 2, stride=2).numpy()
    assert np.allclose(out2, ref[..., ::2], atol=1e-6)


def test_linear_warp_borders():
    f = torch.arange(4, dtype=torch.float32).view(1, 1, 4, 1) + 1.0    # 1,2,3,4
    u = torch.tensor([-0.5, 0.0, 0.5, 1.5]).view(1, 1, 4, 1)
    y = T.linear_warp(f, u).view(-1)
    # x=0: cx=-0.5 -> x0=-1 (masked), x1=0 weight 0.5 -> 0.5 ; x=3: cx=4.5 -> both outside -> 0
    assert torch.allclose(y, torch.tensor([0.5, 2.0, 3.5, 0.0]))
    # image warp clamps instead of masking
    z = T.warp_image(f, -u).view(-1)
    assert torch.allclose(z, torch.tensor([1.0, 2.0, 3.5, 4.0]))


def test_param_table():
    shapes = param_shapes()
    assert sum(int(np.prod(s)) for s in shapes.values()) == 3826070        # SURVEY §8(a) a15
    groups = mad_groups_full()
    sizes = [sum(int(np.prod(shapes[n])) for n in g) for g in groups]
    assert sizes == [1112801, 745185, 588449, 468577, 911058]


def test_golden_snapshot():
    torch.set_num_threads(1)
    g = np.load(GOLDEN)
    left = g['left'].astype(np.float32); right = g['right'].astype(np.float32)
    params = init_params(seed=42)
    net = MadNetOracle(params)
    disps, layers = net.forward(left, right)
    for i, d in enumerate(disps):
        ref = g['disp%d' % i]
        assert np.abs(d.numpy() - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max())
    loss = float(T.reprojection_loss(disps[-1], torch.tensor(left), torch.tensor(right)))
    assert abs(loss - float(g['full_loss'])) < 1e-5
    ad = OracleAdapter(params, mode='MAD')
    o = ad.step(left, right, 2)
    assert abs(o['train_loss'] - float(g['MAD2:train_loss'])) < 1e-5
    for n, gr in o['grads'].items():
        if n.endswith('weights'):
            ref = float(g['MAD2:gnorm:' + n])
            assert abs(np.sqrt((gr.astype(np.float64) ** 2).sum()) - ref) <= 1e-3 * ref + 1e-9


def test_fp64_cross_check():
    g = np.load(GOLDEN)
    left = g['left'].astype(np.float32); right = g['right'].astype(np.float32)
    params = init_params(seed=42)
    d32, _ = MadNetOracle(params).forward(left, right)
    d64, _ = MadNetOracle(params, dtype=torch.float64).forward(left, right)
    for a, b in zip(d32, d64):
        assert float((a.double() - b).abs().max()) <= 1e-4 * max(1.0, float(b.abs().max()))


# ---------------------------------------------------------------------------------------------------
# vectors produced by the REFERENCE'S OWN graph code (Nets/*.py, Losses/loss_factory.py, Data_utils/preprocessing.py
# imported unmodified from /root/reference and executed over oracle/tf1_shim.py by oracle/run_reference_graph.py in the
# build container; fixtures committed under tests/golden/).  They pin the oracle's wiring, warps, losses, variable
# naming and MAD variable lists to the reference; conv SAME padding / legacy resize / crop_or_pad kernels are shared
# with the shim and therefore NOT independently pinned (DESIGN.md section 2).
# ---------------------------------------------------------------------------------------------------
REF_MADNET = os.path.join(os.path.dirname(__file__), 'golden', 'reference_graph_madnet_64x128.npz')
REF_DISPNET = os.path.join(os.path.dirname(__file__), 'golden', 'reference_graph_dispnet_64x128.npz')


def _sub(a, n=4096):
    a = np.asarray(a).ravel()                       # same deterministic subsample as oracle/run_reference_graph.py:sub
    return a[::max(1, a.size // n)]


def _rel(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def test_oracle_forward_matches_reference_graph_madnet():
    import json
    g = np.load(REF_MADNET)
    left = g['left'].astype(np.float32); right = g['right'].astype(np.float32)
    params = init_params(seed=42)
    assert list(g['variable_names']) == list(param_shapes().keys())            # creation order == checkpoint order
    assert [tuple(json.loads(s)) for s in g['variable_shapes']] == [tuple(v) for v in param_shapes().values()]
    disps, layers = MadNetOracle(params).forward(left, right)
    assert len(disps) == 6
    for i, d in enumerate(disps):
        assert d.shape == g['disp%d' % i].shape
        assert _rel(d.numpy(), g['disp%d' % i]) < 5e-5, i
    for k in [k for k in g.files if k.startswith('layer:')]:
        assert _rel(layers[k[6:]].numpy(), g[k]) < 5e-5, k
    loss = float(T.reprojection_loss(disps[-1], torch.tensor(left), torch.tensor(right)))
    assert abs(loss - float(g['full_loss'])) < 2e-6
    # what StereoNet.get_variables returns in the reference (captured when the layer is created, Stereo_net.py:63-67)
    gv = json.loads(str(g['get_variables']))
    assert gv['left/conv1'] == ['model/gc-read-pyramid/conv1/weights:0', 'model/gc-read-pyramid/conv1/biases:0']
    assert gv['right/conv1'] == [] and gv['rescaled_prediction'] == []
    assert len(gv['final_disp']) == 98


def test_oracle_mad_and_full_steps_match_reference_graph():
    g = np.load(REF_MADNET)
    left = g['left'].astype(np.float32); right = g['right'].astype(np.float32)
    params = init_params(seed=42)
    groups = mad_groups_full()
    for k in range(5):
        out = OracleAdapter(params, mode='MAD', lr=1e-4).step(left, right, k)
        assert abs(out['train_loss'] - float(g['mad%d_loss' % k])) < 2e-6, k
        ref_vars = set(g['mad%d_vars' % k]) - set(g['mad%d_none' % k])
        assert set(out['grads']) == ref_vars, k                                 # the reference's var_list for module k
        assert set(groups[k]) == ref_vars, k
        for key in [x for x in g.files if x.startswith('mad%d_grad:' % k)]:
            assert _rel(_sub(out['grads'][key.split(':', 1)[1]]), g[key]) < 2e-4, key
    out = OracleAdapter(params, mode='FULL', lr=1e-4).step(left, right, 0)
    assert abs(out['train_loss'] - float(g['full_mode_loss'])) < 2e-6
    for key in [x for x in g.files if x.startswith('full_grad:')]:
        assert _rel(_sub(out['grads'][key.split(':', 1)[1]]), g[key]) < 2e-4, key


def test_oracle_dispnet_matches_reference_graph():
    from oracle.dispnet import DispNetOracle, DispNetAdapter, init_params as dinit, param_shapes as dshapes
    g = np.load(REF_DISPNET)
    left = g['left'].astype(np.float32); right = g['right'].astype(np.float32)
    p = dinit(seed=7)
    assert list(g['variable_names']) == list(dshapes().keys())
    disps, _ = DispNetOracle(p).forward(left, right)
    assert len(disps) == 7
    for i, d in enumerate(disps):
        assert _rel(d.numpy(), g['disp%d' % i]) < 5e-5, i
    out = DispNetAdapter(p, mode='FULL').step(left, right)
    assert abs(out['train_loss'] - float(g['full_loss'])) < 2e-6
    for key in [x for x in g.files if x.startswith('full_grad:')]:
        assert _rel(_sub(out['grads'][key.split(':', 1)[1]]), g[key]) < 2e-4, key


def test_oracle_matches_reference_graph_at_padded_size():
    """100x200 is not a multiple of 64: the reference's pad_image (REFLECT) and the crop back in _make_disp run as written."""
    g = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'reference_graph_madnet_100x200.npz'))
    left = g['left'].astype(np.float32); right = g['right'].astype(np.float32)
    params = init_params(seed=42)
    disps, layers = MadNetOracle(params).forward(left, right)
    for i, d in enumerate(disps):
        assert tuple(d.shape) == (1, 100, 200, 1)
        assert _rel(d.numpy(), g['disp%d' % i]) < 5e-5, i
    assert _rel(layers['final_disp'].numpy(), g['layer:final_disp']) < 5e-5
    assert abs(float(T.reprojection_loss(disps[-1], torch.tensor(left), torch.tensor(right))) - float(g['full_loss'])) < 2e-6
    for k in range(5):
        out = OracleAdapter(params, mode='MAD', lr=1e-4).step(left, right, k)
        assert abs(out['train_loss'] - float(g['mad%d_loss' % k])) < 2e-6, k


def test_oracle_batch_equals_single_frames():
    """The batch-N reference of the GPU tests (and of N ranks x 1 frame in data-parallel runs): the oracle at batch 3 gives
    the per-frame disparities of three batch-1 runs, and its loss -- a mean over the batch -- is the mean of theirs.
    (torch's CPU convolutions choose their blocking by batch size, so fp32 sums are reordered: ~1e-6 relative.)"""
    from madstereo.synthetic import make_pair
    from oracle.dispnet import DispNetOracle, init_params as dinit
    torch.set_num_threads(1)
    left, right, _ = make_pair(64, 128, seed=3, batch=3)
    for net in (MadNetOracle(init_params(seed=42)), DispNetOracle(dinit(seed=7))):
        disps, _ = net.forward(left, right)
        loss = float(T.reprojection_loss(disps[-1], torch.tensor(left), torch.tensor(right)))
        losses = []
        for b in range(3):
            lb, rb = left[b:b + 1], right[b:b + 1]
            d1, _ = net.forward(lb, rb)
            for i, (d, r) in enumerate(zip(disps, d1)):
                assert d.shape[0] == 3 and _rel(d[b:b + 1].numpy(), r.numpy()) < 1e-5, (type(net).__name__, b, i)
            losses.append(float(T.reprojection_loss(d1[-1], torch.tensor(lb), torch.tensor(rb))))
        assert abs(loss - np.mean(losses)) <= 1e-6 * abs(loss), (type(net).__name__, loss, losses)
