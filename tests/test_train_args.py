"""python -m esac_b200.train on the host: train_esac.py's options and defaults, the file names it reads and writes, the
epoch count, the log line, and the refusal of model files that do not fit the environment."""
import os

import pytest
import torch

from esac_b200 import train
from esac_b200.data import ClusterDraws, RoomDraws
from oracle import expert_oracle as XO
from oracle import gating_oracle as GO

# train_esac.py:20-63: long name, short name, default
OPTIONS = [("hypotheses", "-hyps", 256), ("threshold", "-t", 10), ("inlieralpha", "-ia", 100), ("inlierbeta", "-ib", 0.5),
           ("maxreprojection", "-maxr", 100), ("learningrate", "-lr", 0.000001), ("iterations", "-iter", 50000),
           ("weightrot", "-wr", 1.0), ("weighttrans", "-wt", 100.0), ("losscut", "-lc", 100.0),
           ("clusters", "-c", -1), ("maxexperts", "-maxe", -1), ("expertselection", "-es", False),
           ("session", "-sid", ""), ("refined", "-ref", False)]


def test_options_are_train_esacs():
    opt = vars(train.options([]))
    assert opt == dict({name: default for name, _, default in OPTIONS}, seed=0)
    values = {"hypotheses": "64", "threshold": "7.5", "inlieralpha": "50", "inlierbeta": "0.25", "maxreprojection": "60",
              "learningrate": "0.001", "iterations": "12", "weightrot": "2", "weighttrans": "50", "losscut": "30",
              "clusters": "4", "maxexperts": "2", "session": "s"}
    short, long = [], []
    for name, flag, default in OPTIONS:
        if isinstance(default, bool):
            short.append(flag)
            long.append("--" + name)
        else:
            short += [flag, values[name]]
            long += ["--" + name, values[name]]
    a, b = train.options(short + ["--seed", "5"]), train.options(long + ["--seed", "5"])
    assert vars(a) == vars(b)
    assert (a.hypotheses, a.threshold, a.learningrate, a.clusters, a.maxexperts, a.session, a.seed) == \
        (64, 7.5, 0.001, 4, 2, "s", 5)
    assert a.expertselection and a.refined


@pytest.mark.parametrize("argv", [["-iter", "0"], ["-hyps", "0"]])
def test_options_refuse_empty_runs(argv):
    with pytest.raises(SystemExit):
        train.options(argv)


def test_help_states_the_departures(capsys):
    with pytest.raises(SystemExit):
        train.options(["--help"])
    text = " ".join(capsys.readouterr().out.split())
    for words in ("one line per epoch", "counter-based generator", "TF32", "saved once more after the last iteration"):
        assert words in text
    for words in ("one line per epoch", "counter-based generator", "TF32", "saved once more after the last iteration"):
        assert words in " ".join(train.__doc__.split())


@pytest.mark.parametrize("flags, model, log, gating, expert1", [
    ([], "esac_sid.net", "log_esac_sid.txt", "./gating_sid.net", "./expert_e1_sid.net"),
    (["-es"], "es_sid.net", "log_es_sid.txt", "./gating_sid.net", "./expert_e1_sid.net"),
    (["-ref"], "esac_sid.net", "log_esac_sid.txt", "./gating_sid.net", "./expert_e1_sid_refined.net"),
    (["-es", "-ref"], "es_sid.net", "log_es_sid.txt", "./gating_sid.net", "./expert_e1_sid_refined.net"),
])
def test_file_names(flags, model, log, gating, expert1):
    opt = train.options(flags + ["-sid", "sid"])
    assert train.output_files(opt) == (model, log)
    g, ex = train.input_files(opt, 3)
    assert g == gating and len(ex) == 3 and ex[1] == expert1


def test_file_names_without_a_session():
    opt = train.options([])
    assert train.output_files(opt) == ("esac_.net", "log_esac_.txt")
    assert train.input_files(opt, 1) == ("./gating_.net", ["./expert_e0_.net"])


def test_epochs_count_the_draws():
    rooms = RoomDraws([3, 4, 5], training=True)
    assert len(rooms) == 1000                                  # RoomDataset's training epoch, whatever the image count
    assert train.epochs(50000, len(rooms)) == 50
    assert train.epochs(1, len(rooms)) == 1 and train.epochs(1001, len(rooms)) == 2
    clusters = ClusterDraws(7)
    assert train.epochs(20, len(clusters)) == 3 and train.epochs(21, len(clusters)) == 3 and train.epochs(22, 7) == 4


def test_log_line_is_train_esacs():
    assert train.log_line(0, 12.5) == "0 12.500000 \n"
    assert train.log_line(41, 0.1234567) == "41 0.123457 \n"


def write_inputs(root, E, capacity, refined=False, session="syn"):
    suffix = "_refined" if refined else ""
    torch.save(GO.kaiming_state_dict(1, E, capacity), root / f"gating_{session}.net")
    for e in range(E):
        torch.save(XO.kaiming_state_dict(2 + e, mean=(float(e), 0.0, 1.0)), root / f"expert_e{e}_{session}{suffix}.net")


def load(root, argv, E, capacity):
    prev = os.getcwd()
    os.chdir(root)
    try:
        return train.load_networks(train.options(argv), E, capacity, "cpu")
    finally:
        os.chdir(prev)


def test_loads_the_individual_files(tmp_path):
    write_inputs(tmp_path, 3, 1)
    gating, experts = load(tmp_path, ["-sid", "syn"], 3, 1)
    assert len(experts) == 3 and gating.capacity == 1
    for e, m in enumerate(experts):
        want = torch.load(tmp_path / f"expert_e{e}_syn.net")
        assert all(torch.equal(m.state_dict()[k], v) for k, v in want.items())
    write_inputs(tmp_path, 2, 2, refined=True, session="cl")
    gating, experts = load(tmp_path, ["-sid", "cl", "-ref"], 2, 2)
    assert gating.capacity == 2 and len(experts) == 2


def test_refuses_files_that_do_not_fit(tmp_path):
    write_inputs(tmp_path, 3, 1)
    with pytest.raises(RuntimeError, match=r"gating_syn\.net: the gating network has 3 experts at capacity 1; the "
                                           r"environment needs 4 at capacity 1"):
        load(tmp_path, ["-sid", "syn"], 4, 1)
    with pytest.raises(RuntimeError, match=r"gating_syn\.net: .* 3 experts at capacity 1; .* needs 3 at capacity 2"):
        load(tmp_path, ["-sid", "syn"], 3, 2)
    with pytest.raises(FileNotFoundError, match=r"expert_e0_syn_refined\.net"):
        load(tmp_path, ["-sid", "syn", "-ref"], 3, 1)

    sd = torch.load(tmp_path / "expert_e1_syn.net")
    sd["conv9.weight"] = sd.pop("conv2.weight")
    torch.save(sd, tmp_path / "expert_e1_syn.net")
    with pytest.raises(RuntimeError, match=r"expert_e1_syn\.net: state dict keys differ from Expert's \(missing "
                                           r"\['conv2.weight'\], unexpected \['conv9.weight'\]\)"):
        load(tmp_path, ["-sid", "syn"], 3, 1)

    write_inputs(tmp_path, 3, 1)
    gsd = torch.load(tmp_path / "gating_syn.net")
    gsd["fc2.bias"] = torch.zeros(5)
    torch.save(gsd, tmp_path / "gating_syn.net")
    with pytest.raises(RuntimeError, match=r"gating_syn\.net: fc2.bias must be \[64\], got \[5\]"):
        load(tmp_path, ["-sid", "syn"], 3, 1)
    del gsd["fc3.weight"]
    torch.save(gsd, tmp_path / "gating_syn.net")
    with pytest.raises(RuntimeError, match=r"gating_syn\.net: .*missing \['fc3.weight'\]"):
        load(tmp_path, ["-sid", "syn"], 3, 1)


def test_saves_the_ensemble_layout(tmp_path):
    write_inputs(tmp_path, 2, 1)
    gating, experts = load(tmp_path, ["-sid", "syn"], 2, 1)
    train.save_model(str(tmp_path / "esac_syn.net"), gating, experts)
    sds = torch.load(tmp_path / "esac_syn.net")
    assert isinstance(sds, list) and len(sds) == 3
    assert set(sds[0]) == set(GO.state_dict_shapes(2, 1)) and all(set(sd) == set(XO.state_dict_shapes()) for sd in sds[1:])
