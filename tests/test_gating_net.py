"""The gating network without a GPU (esac_b200/gating_net.py, oracle/gating_oracle.py): the state dict's keys, shapes and
dtypes, every rejected argument of forward_async, the C ABI's sizes, the packed layout, and the float64 oracle against the
restated Gating module."""
import numpy as np
import pytest
import torch

from esac_b200.gating_net import GatingNet, network_size, state_dict_shapes
from oracle import gating_oracle as O


def sd(E=7, c=1, seed=0):
    return O.kaiming_state_dict(seed, E, c)


@pytest.mark.parametrize("E, c", [(7, 1), (50, 2), (1, 1)])
def test_state_dict_shapes_are_gatings(E, c):
    want = {k: tuple(v.shape) for k, v in O.make_gating_class()(E, c).state_dict().items()}
    assert state_dict_shapes(E, c) == want and list(state_dict_shapes(E, c)) == list(want)
    assert network_size(sd(E, c)) == (E, c)


@pytest.mark.parametrize("edit, match", [
    (lambda d: d.pop("fc2.bias"), "gating: state dict keys differ from Gating's \\(missing \\['fc2.bias'\\]"),
    (lambda d: d.pop("fc3.weight"), "missing \\['fc3.weight'\\]"),
    (lambda d: d.pop("conv4.weight"), "missing \\['conv4.weight'\\]"),
    (lambda d: d.__setitem__("fc4.weight", torch.zeros(7, 64, 1, 1)), "unexpected \\['fc4.weight'\\]"),
    (lambda d: d.__setitem__("conv2.weight", torch.zeros(16, 8, 1, 1)), "gating: conv2.weight must be \\[16, 8, 3, 3\\]"),
    (lambda d: d.__setitem__("fc3.bias", torch.zeros(6)), "fc3.bias must be \\[7\\]"),
    (lambda d: d.__setitem__("res1_conv2.weight", torch.zeros(64, 64, 3, 3)), "res1_conv2.weight must be \\[64, 64, 1, 1\\]"),
    (lambda d: d.__setitem__("fc1.weight", torch.zeros(256, 64, 1, 1)), "fc1.weight must be \\[64, 64, 1, 1\\]"),
    (lambda d: d.__setitem__("conv4.weight", torch.zeros(96, 32, 3, 3)), "conv4.weight must be \\[64, 32, 3, 3\\] \\(capacity 1\\)"),
    (lambda d: d.__setitem__("conv4.weight", torch.zeros(64, 32)), "conv4.weight must be a 4-d"),
    (lambda d: d.__setitem__("fc3.weight", torch.zeros(1025, 64, 1, 1)), "1025 experts, outside \\[1, 1024\\]"),
    (lambda d: d.__setitem__("conv1.bias", torch.zeros(8, dtype=torch.int64)), "conv1.bias must be a floating-point tensor"),
    (lambda d: d.__setitem__("conv1.bias", [0.0] * 8), "conv1.bias must be a floating-point tensor"),
])
def test_state_dict_rejected(edit, match):
    bad = sd()
    edit(bad)
    with pytest.raises(RuntimeError, match=match):
        GatingNet(bad, "cuda")


def test_capacity_two_shapes_are_checked():
    bad = sd(10, 2)
    bad["fc2.weight"] = torch.zeros(128, 128, 1, 1)
    with pytest.raises(RuntimeError, match="fc2.weight must be \\[256, 256, 1, 1\\]"):
        GatingNet(bad, "cuda")
    with pytest.raises(RuntimeError, match="CUDA device"):
        GatingNet(sd(), "cpu")


def stub(E=7, c=1):
    """A GatingNet whose weights were never packed: enough for the checks that precede any device work."""
    g = object.__new__(GatingNet)
    g.E, g.capacity, g.device, g.packed, g.workspace, g.frozen = E, c, torch.device("cuda", 0), None, None, False
    return g


@pytest.mark.parametrize("case, match", [
    ("image_float64", "expected scalar type Float but found Double \\(image\\)"),
    ("image_rank", "expected 4 dims but tensor has 3 \\(image\\)"),
    ("image_channels", "image must be \\[B,3,H,W\\]"),
    ("image_numpy", "torch CUDA tensors only \\(image is a ndarray\\)"),
    ("image_noncontig", "image must be contiguous"),
    ("log_half", "expected scalar type Float but found Half \\(out_log_probs\\)"),
    ("log_shape", "out_log_probs must be a contiguous \\[2, 7\\] tensor"),
    ("log_batch", "out_log_probs must be a contiguous \\[2, 7\\] tensor"),
    ("log_noncontig", "out_log_probs must be a contiguous"),
    ("log_numpy", "torch CUDA tensors only \\(out_log_probs is a ndarray\\)"),
    ("probs_shape", "out_probs must be a contiguous \\[2, 7\\] tensor"),
    ("probs_double", "expected scalar type Float but found Double \\(out_probs\\)"),
    ("cpu", "takes CUDA tensors only \\(image is on the CPU\\)"),
])
def test_forward_async_rejected(case, match):
    image, log_p, probs = torch.zeros(2, 3, 16, 24), torch.zeros(2, 7), None
    if case == "image_float64":
        image = image.double()
    elif case == "image_rank":
        image = image[0]
    elif case == "image_channels":
        image = torch.zeros(2, 4, 16, 24)
    elif case == "image_numpy":
        image = image.numpy()
    elif case == "image_noncontig":
        image = torch.zeros(2, 3, 24, 16).transpose(2, 3)
    elif case == "log_half":
        log_p = log_p.half()
    elif case == "log_shape":
        log_p = torch.zeros(2, 6)
    elif case == "log_batch":
        log_p = torch.zeros(1, 7)
    elif case == "log_noncontig":
        log_p = torch.zeros(7, 2).t()
    elif case == "log_numpy":
        log_p = log_p.numpy()
    elif case == "probs_shape":
        probs = torch.zeros(2, 8)
    elif case == "probs_double":
        probs = torch.zeros(2, 7, dtype=torch.float64)
    with pytest.raises(RuntimeError, match=match):
        stub().forward_async(image, log_p, probs)


def test_reserve_rejects_sizes():
    with pytest.raises(RuntimeError, match="sizes must be positive"):
        stub().reserve(1, 0, 16)
    with pytest.raises(RuntimeError, match="outside the supported range"):
        stub().workspace_bytes(65536, 16, 16)
    with pytest.raises(RuntimeError, match="outside the supported range"):
        stub().workspace_bytes(1, 16, 8193)


def test_frozen_workspace_does_not_grow():
    g = stub()
    g.workspace, g.frozen = torch.empty(g.workspace_bytes(1, 16, 16), dtype=torch.uint8), True
    g.reserve(1, 16, 16)
    with pytest.raises(RuntimeError, match="a captured graph already uses"):
        g.reserve(2, 16, 16)


def test_packed_and_workspace_sizes(lib):
    for E in (1, 7, 19, 50, 1024):
        for c in (1, 2):
            assert lib.esacb200_gating_packed_floats(E, c) == O.packed_floats(E, c)
    for E, c in ((0, 1), (1025, 1), (7, 0), (7, 3)):
        assert lib.esacb200_gating_packed_floats(E, c) == -1
    # 480x640, capacity 2: conv3's 32 channels at /4, two 128-channel maps at /8, 38 chunks of 128 cells x 128 sums;
    # a 256-byte header of ints for the image list
    per_image = 32 * 120 * 160 + 2 * 128 * 60 * 80 + 38 * 128
    assert lib.esacb200_gating_workspace_bytes(3, 10, 2, 480, 640) == 256 + 3 * 4 * per_image
    assert lib.esacb200_gating_workspace_bytes(1, 7, 1, 1, 1) == 256 + 4 * (64 + 64 + 64 + 64)
    for args in ((0, 7, 1, 8, 8), (65536, 7, 1, 8, 8), (1, 0, 1, 8, 8), (1, 7, 3, 8, 8), (1, 7, 1, 8193, 8),
                 (1, 7, 1, 8, 0)):
        assert lib.esacb200_gating_workspace_bytes(*args) == -1


@pytest.mark.parametrize("E, c", [(7, 1), (10, 2)])
def test_pack_layout_round_trips(E, c):
    weights = sd(E, c, seed=3)
    packed = O.pack(weights, c)
    back = O.unpack(packed, E, c)
    assert list(back) == list(state_dict_shapes(E, c))
    for k, v in weights.items():
        want = v.numpy()
        if k.split(".")[0] in O.GEMM and k.endswith(".weight"):
            want = O.tf32(want)
        assert np.array_equal(back[k], want), k
    # the front end reads a tap's output channels contiguously, the GEMM layers a tap's input channels, the head an input's
    # outputs
    segs, _ = O._segments(E, c)
    w1 = weights["conv1.weight"].numpy()
    assert packed[segs[0][1] + (1 * 3 + 2) * 3 * 8 + 1 * 8 + 5] == w1[5, 1, 1, 2]
    w4 = weights["conv4.weight"].numpy()
    assert packed[segs[3][1] + ((3 * 3 + 2) * 3 + 1) * 32 + 9] == O.tf32(w4[3, 9, 2, 1])
    w9 = weights["fc3.weight"].numpy()
    assert packed[segs[9][1] + 11 * E + 4] == w9[4, 11, 0, 0]


@pytest.mark.parametrize("E, c, hw", [(7, 1, (37, 53)), (50, 2, (24, 40)), (1, 1, (9, 8)), (19, 1, (64, 80))])
def test_oracle_equals_gating_module(E, c, hw):
    weights = sd(E, c, seed=E + c)
    g = torch.Generator().manual_seed(5)
    image = torch.randn((2, 3) + hw, generator=g, dtype=torch.float64)
    module = O.make_gating_class()(E, c).double()
    module.load_state_dict(weights)
    with torch.no_grad():
        want = module(image)
    got = O.forward(image, weights, c)
    assert got.shape == (2, E) and got.dtype == torch.float64
    assert float((got - want).abs().max()) <= 1e-12


def test_cpu_has_no_fallback():
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(RuntimeError):
        GatingNet(sd(), "cuda")


# test_esac.py's options (test_esac.py:15-59): long name, short name, default
TEST_ESAC_OPTIONS = [("model", "-m", ""), ("testinit", "-tinit", False), ("testrefined", "-tref", False),
                     ("hypotheses", "-hyps", 256), ("threshold", "-t", 10), ("inlieralpha", "-ia", 100),
                     ("inlierbeta", "-ib", 0.5), ("maxreprojection", "-maxr", 100), ("rotthreshold", "-rt", 5),
                     ("transthreshold", "-tt", 5), ("expertselection", "-es", False), ("oracleselection", "-os", False),
                     ("clusters", "-c", -1), ("session", "-sid", "")]


def test_localize_options_are_test_esacs():
    from esac_b200 import localize
    opt = vars(localize.options([]))
    assert opt == {**{name: default for name, _, default in TEST_ESAC_OPTIONS}, "seed": 0}
    given = {"model": "a.net", "hypotheses": 64, "threshold": 4.5, "inlieralpha": 50.0, "inlierbeta": 0.25,
             "maxreprojection": 80.0, "rotthreshold": 2.0, "transthreshold": 3.0, "clusters": 10, "session": "s"}
    argv = [a for name, short, _ in TEST_ESAC_OPTIONS if name in given for a in (short, str(given[name]))]
    argv += ["-tinit", "-tref", "-es", "--seed", "9"]
    opt = vars(localize.options(argv))
    assert opt == {**given, "testinit": True, "testrefined": True, "expertselection": True, "oracleselection": False,
                   "seed": 9}
    long = [a for name, _, _ in TEST_ESAC_OPTIONS if name in given for a in ("--" + name, str(given[name]))]
    assert vars(localize.options(long + ["--testinit", "--testrefined", "--expertselection", "--seed", "9"])) == opt
    with pytest.raises(SystemExit):
        localize.options(["-c", "4", "-os"])     # a clustered environment has no ground-truth expert


@pytest.mark.parametrize("flags, session, files", [
    ([], "sid", ("ensemble", "esac_sid.net")),
    (["-es"], "es_sid", ("ensemble", "es_sid.net")),
    (["-os"], "os_sid", ("ensemble", "esac_sid.net")),
    (["-es", "-os"], "os_es_sid", ("ensemble", "es_sid.net")),
    (["-m", "my.net", "-es"], "es_sid", ("ensemble", "my.net")),
    (["-tinit"], "init_sid", ("individual", "./gating_sid.net", ["./expert_e0_sid.net", "./expert_e1_sid.net"])),
    (["-tref"], "ref_sid", ("individual", "./gating_sid.net",
                            ["./expert_e0_sid_refined.net", "./expert_e1_sid_refined.net"])),
    (["-tinit", "-tref", "-es"], "es_ref_init_sid", ("individual", "./gating_sid.net",
                                                     ["./expert_e0_sid_refined.net", "./expert_e1_sid_refined.net"])),
])
def test_localize_session_prefixes_and_model_files(flags, session, files):
    """test_esac.py:88-114 and expert_ensemble.py:94-112: the model default depends on -es only, the individual files on
    the unprefixed session (the refined experts add _refined, the gating does not), the output prefixes stack in the
    order init_, ref_, es_, os_."""
    from esac_b200 import localize
    opt = localize.options(flags + ["-sid", "sid"])
    assert localize.model_files(opt, 2) == files
    assert localize.output_session(opt) == session


def test_localize_strips_file_names():
    from esac_b200.localize import strip_file_name
    assert strip_file_name("/d/chess/test/rgb/frame-000001.color.png") == "frame-000001.color.png"
    assert strip_file_name("aachen/test/rgb/query_night_nexus5x_IMG_1.jpg") == "IMG_1.jpg"
    assert strip_file_name("db_12.jpg") == "12.jpg"
