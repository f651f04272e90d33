"""Which backward a call trains through, without a GPU: api._train_path over every precision x set_backward x gradients needed x
fine network (none, agreeing or disagreeing with the coarse one on use_viewdirs), for the drop-in calls (render, render_rays)
and for FusedTrainStep, pinned as an explicit table; the refusals that public calls make before any launch; and the entry
points each tensor-core training path names."""
import itertools

import pytest
import torch

PRECISIONS = ("tc_fp16", "tc_split", "fp32")
BACKWARDS = ("tc", "exact", "tc_split")
FINE = ("none", "agree", "disagree")

# refusals: the words each message contains
PREC = "set_backward('tc_split') needs precision tc_split (precision is {precision}): call set_precision('tc_split') or set_backward('tc')"
VIEWS = "set_backward('tc_split') needs the coarse and fine networks to agree on use_viewdirs"
FUSED = "FusedTrainStep runs the tensor-core path (set_precision('tc_fp16'), or set_precision('tc_split') with set_backward('tc_split'))"
FUSED_VIEWS = "FusedTrainStep: coarse and fine networks must agree on use_viewdirs (they share the ray batch)"

# (precision, backward) -> (path with no fine network or an agreeing one, path with a disagreeing one) of a call that needs gradients
DROPIN = {
    ("tc_fp16", "tc"): ("fp16", "exact"),             # disagreeing networks fall back to the exact backward
    ("tc_fp16", "exact"): ("exact", "exact"),
    ("tc_fp16", "tc_split"): (PREC, PREC),
    ("tc_split", "tc"): ("exact", "exact"),
    ("tc_split", "exact"): ("exact", "exact"),
    ("tc_split", "tc_split"): ("split", VIEWS),
    ("fp32", "tc"): ("exact", "exact"),
    ("fp32", "exact"): ("exact", "exact"),
    ("fp32", "tc_split"): (PREC, PREC),
}
FUSED_STEP = {
    ("tc_fp16", "tc"): ("fp16", FUSED_VIEWS),
    ("tc_fp16", "exact"): ("fp16", FUSED_VIEWS),       # tc_fp16 trains on fp16 records whatever set_backward says
    ("tc_fp16", "tc_split"): ("fp16", FUSED_VIEWS),
    ("tc_split", "tc"): (FUSED, FUSED),
    ("tc_split", "exact"): (FUSED, FUSED),
    ("tc_split", "tc_split"): ("split", FUSED_VIEWS),
    ("fp32", "tc"): (FUSED, FUSED),
    ("fp32", "exact"): (FUSED, FUSED),
    ("fp32", "tc_split"): (FUSED, FUSED),
}


@pytest.fixture(scope="module")
def nb():
    import __graft_entry__ as ge
    ge.build()
    import nerf_pytorch_b200
    return nerf_pytorch_b200


@pytest.fixture
def modes(nb):
    yield
    nb.set_precision("tc_fp16")
    nb.set_backward("tc")


def _net(nb, viewdirs):
    return nb.NeRF(D=2, W=32, input_ch=63, input_ch_views=27 if viewdirs else 0, output_ch=5 if viewdirs else 4, skips=[4],
                   use_viewdirs=viewdirs)


def _nets(nb, fine):
    return _net(nb, True), {"none": None, "agree": _net(nb, True), "disagree": _net(nb, False)}[fine]


def _expect(table, precision, backward, fine, want_grad=True):
    if not want_grad:
        return None
    return table[(precision, backward)][fine == "disagree"].format(precision=precision)


def _taken(nb, precision, backward, want_grad, net_c, net_f, fused=False):
    """The path api._train_path picks ("fp16", "split", "exact" or None), or its refusal's message."""
    from nerf_pytorch_b200 import api
    try:
        path = api._train_path(precision, backward, want_grad, net_c, net_f, fused=fused)
    except RuntimeError as e:
        return str(e)
    return {id(api._TC_FP16): "fp16", id(api._TC_SPLIT): "split"}.get(id(path), path)


@pytest.mark.parametrize("precision,backward,want_grad,fine", list(itertools.product(PRECISIONS, BACKWARDS, (True, False), FINE)))
def test_dropin_path(nb, precision, backward, want_grad, fine):
    assert _taken(nb, precision, backward, want_grad, *_nets(nb, fine)) == _expect(DROPIN, precision, backward, fine, want_grad)


@pytest.mark.parametrize("precision,backward,fine", list(itertools.product(PRECISIONS, BACKWARDS, FINE)))
def test_fused_step_path(nb, precision, backward, fine):
    assert _taken(nb, precision, backward, True, *_nets(nb, fine), fused=True) == _expect(FUSED_STEP, precision, backward, fine)


def test_refusals_without_networks(nb):
    """Without networks (render() given modules that are not NeRF) the decision is that of a call without a fine network."""
    for precision, backward in itertools.product(PRECISIONS, BACKWARDS):
        assert _taken(nb, precision, backward, True, None, None) == _expect(DROPIN, precision, backward, "none")


def test_path_entries_are_library_symbols(nb):
    from nerf_pytorch_b200 import _lib, api
    for path, image in ((api._TC_FP16, nb.NeRF.packed), (api._TC_SPLIT, nb.NeRF.packed_split_train)):
        assert path.image is image
        names = [v for k, v in path._asdict().items() if k != "image" and v is not None]
        assert len(names) == len(set(names))
        for name in names:
            assert name in _lib.SIGNATURES, name
    # the split path takes NerfOutGrads seeds only; fp16 has an rgb-only entry for one pass and for both
    assert api._TC_SPLIT.march_bwd_rgb is None and api._TC_SPLIT.bwd_rgb is None
    assert api._TC_FP16.march_bwd_rgb and api._TC_FP16.bwd_rgb
    assert not set(api._TC_FP16._asdict().values()) & set(api._TC_SPLIT._asdict().values())


# ---- refusals public calls make on the CPU before any launch ----------------------------------------------------------------------

def _render_kwargs(nb, net_c, net_f, N_importance):
    from nerf_pytorch_b200 import api
    q = api._QueryFn(None, None, 1024, 10, 4, 0)
    return dict(network_fn=net_c, network_fine=net_f, network_query_fn=q, N_samples=8, N_importance=N_importance, perturb=0.,
                white_bkgd=False, raw_noise_std=0., use_viewdirs=True, ndc=False, near=2., far=6.)


@pytest.mark.parametrize("precision", ["tc_fp16", "fp32"])
@pytest.mark.parametrize("fine", FINE)
def test_render_refuses_split_backward_in_other_precisions(nb, modes, precision, fine):
    net_c, net_f = _nets(nb, fine)
    nb.set_precision(precision)
    nb.set_backward("tc_split")
    K = [[100., 0., 50.], [0., 100., 50.], [0., 0., 1.]]
    rays = (torch.zeros(4, 3), torch.ones(4, 3))
    kw = _render_kwargs(nb, net_c, net_f, 8 if net_f is not None else 0)
    n0 = nb.launch_count()
    with pytest.raises(RuntimeError) as e:
        nb.render(100, 100, K, rays=rays, **kw)
    assert str(e.value) == PREC.format(precision=precision)
    assert nb.launch_count() == n0
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):       # without gradients there is nothing to refuse
        nb.render(100, 100, K, rays=rays, **kw)
    for p in list(net_c.parameters()) + (list(net_f.parameters()) if net_f is not None else []):
        p.requires_grad_(False)
    with pytest.raises(RuntimeError, match="CUDA"):
        nb.render(100, 100, K, rays=rays, **kw)


@pytest.mark.parametrize("precision,backward", list(itertools.product(PRECISIONS, BACKWARDS)))
def test_fused_step_constructor_refusals(nb, modes, precision, backward):
    from nerf_pytorch_b200.trainer import FusedTrainStep
    nb.set_precision(precision)
    nb.set_backward(backward)
    K = [[100., 0., 50.], [0., 100., 50.], [0., 0., 1.]]
    n0 = nb.launch_count()
    with pytest.raises(RuntimeError) as e:
        FusedTrainStep(100, 100, K, 64, _render_kwargs(nb, *_nets(nb, "agree"), 8))
    if FUSED_STEP[(precision, backward)][0] == FUSED:
        assert str(e.value) == FUSED
    else:                                                                   # accepted: the CPU networks are refused next
        assert "CUDA device" in str(e.value)
    with pytest.raises(RuntimeError, match="needs nerf_b200.NeRF networks"):
        FusedTrainStep(100, 100, K, 64, dict(_render_kwargs(nb, None, None, 0), network_fn=torch.nn.Linear(2, 2)))
    assert nb.launch_count() == n0
