"""Tied embeddings (``--tie_embeddings``) without a GPU: flag validation, the initial draws with and without the flag, the tied
model against an fp64 ``nn.Embedding`` + ``nn.LSTM`` + ``F.linear(h, emb.weight, bias)`` model (fixed and ragged lengths, a
carried state), the class-major reference ops, checkpoints, a short training run with eval and generate, and two gloo ranks."""
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch

from lstm_tensorspark_b200 import data as D
from lstm_tensorspark_b200.config import Config
from lstm_tensorspark_b200.models.classifier import SequenceClassifier
from lstm_tensorspark_b200.ops import reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "untied_lm_init.json")


def _cfg(**kw):
    base = dict(hidden_units="16", in_features=16, seq_len=4, batch_size=3, vocab_size=64, next_token=True, init="scaled",
                learn_initial_state=False, device="cpu")
    base.update(kw)
    return Config(**base).validate()


def _model(cfg, seed=7, dtype=None):
    m = SequenceClassifier(cfg, batch_size=cfg.batch_size, device="cpu", generator=torch.Generator().manual_seed(seed))
    if dtype is not None:
        m = m.to(dtype)
        m.set_compute_dtype(dtype)
    return m


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().numpy().tobytes()).hexdigest()


# ---- flags ------------------------------------------------------------------------------------------------------------------
def test_flag_needs_next_token():
    with pytest.raises(ValueError) as ei:
        Config(tie_embeddings=True, vocab_size=64, in_features=16, hidden_units="16", seq_len=4).validate()
    assert "--tie_embeddings" in str(ei.value) and "--next_token" in str(ei.value)


def test_flag_needs_the_embedding_width_to_be_the_top_layer_width():
    with pytest.raises(ValueError) as ei:
        _cfg(tie_embeddings=True, in_features=8)
    for name in ("--tie_embeddings", "--in_features", "--hidden_units"):
        assert name in str(ei.value)
    _cfg(tie_embeddings=True, hidden_units="8,16")                         # only the last layer's width matters


def test_flag_parses_and_defaults_off():
    from lstm_tensorspark_b200.config import parse_args
    cfg = parse_args(["--next_token", "--vocab_size", "64", "--in_features", "16", "--hidden_units", "16", "--seq_len", "4",
                      "--tie_embeddings"])
    assert cfg.tie_embeddings and "TIE_EMBEDDINGS = True" in cfg.params_str()
    assert not Config().tie_embeddings


# ---- parameters and draws ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hidden", ["16", "12,16"])
def test_untied_model_draws_what_it_drew_before(hidden):
    """Hashes of every variable of an untied model, recorded before the flag existed: nothing changes without it."""
    want = json.load(open(GOLDEN))[hidden]
    m = _model(_cfg(hidden_units=hidden))
    got = {k: _sha(v) for k, v in m.named_reference_variables()}
    assert got == want["variables"]
    assert m.build_flat().numel == want["flat_numel"]


@pytest.mark.parametrize("hidden", ["16", "12,16"])
def test_tied_model_keeps_every_draw_and_drops_the_softmax_matrix(hidden):
    untied, tied = _model(_cfg(hidden_units=hidden)), _model(_cfg(hidden_units=hidden, tie_embeddings=True))
    u, t = dict(untied.named_reference_variables()), dict(tied.named_reference_variables())
    assert "Dense1/weights" in u and "Dense1/weights" not in t and set(u) - set(t) == {"Dense1/weights"}
    for k, v in t.items():
        assert torch.equal(v, u[k]), k
    assert tied.head.weights is None and all(p is not tied.head.weights for p in tied.parameters())
    w, class_major = tied.head_weights()
    assert class_major and w is tied.embedding.weights
    H, V = 16, 64
    assert untied.build_flat().numel - tied.build_flat().numel == H * V
    assert all(p.shape != (H, V) for p in tied.flat.params)


# ---- fp64 against nn.Embedding + nn.LSTM + F.linear(h, emb.weight, bias) -------------------------------------------------------
def _torch_lm(m):
    """The same weights in torch modules: the gates of ``w_x`` / ``w_h`` / ``bias`` are interleaved (``reference.lstm_gates``),
    nn.LSTM stacks them as (i, f, g, o)."""
    emb = torch.nn.Embedding.from_pretrained(m.embedding.weights.detach().clone(), freeze=False)
    layers = m.rnn.layers
    lstm = torch.nn.LSTM(layers[0].w_x.shape[1], layers[0].w_h.shape[1], num_layers=len(layers), dtype=torch.float64)
    order = [ref.GATE_I, ref.GATE_F, ref.GATE_G, ref.GATE_O]
    perm = lambda w: torch.cat([w[g::4] for g in order])
    with torch.no_grad():
        for l, layer in enumerate(layers):
            getattr(lstm, f"weight_ih_l{l}").copy_(perm(layer.w_x.detach()))
            getattr(lstm, f"weight_hh_l{l}").copy_(perm(layer.w_h.detach()))
            getattr(lstm, f"bias_ih_l{l}").copy_(perm(layer.bias.detach()))
            getattr(lstm, f"bias_hh_l{l}").zero_()
    bias = m.head.bias.detach().clone().requires_grad_(True)
    return emb, lstm, bias, perm


def _torch_forward(emb, lstm, bias, x, y, lengths, state):
    B, T = x.shape
    e = emb(x.long())                                                            # [B,T,E]
    hc = None if state is None else tuple(torch.stack(s) for s in zip(*state))
    if lengths is None:
        out, _ = lstm(e.transpose(0, 1), hc)
    else:
        packed = torch.nn.utils.rnn.pack_padded_sequence(e, lengths.long(), batch_first=True, enforce_sorted=False)
        out, _ = lstm(packed, hc)
        out = torch.nn.utils.rnn.pad_packed_sequence(out, total_length=T)[0]
    logits = torch.nn.functional.linear(out.transpose(0, 1), emb.weight, bias)    # [B,T,V]: the table is the softmax matrix
    keep = ref.step_mask(lengths, B, T)
    loss = torch.nn.functional.cross_entropy(logits[keep], y[keep].long())
    return loss, logits


@pytest.mark.parametrize("case", ["fixed", "ragged", "stateful"])
def test_tied_model_equals_the_torch_model_in_fp64(case):
    hidden = "16,16"                                                             # nn.LSTM stacks layers of one width
    cfg = _cfg(hidden_units=hidden, tie_embeddings=True, batch_size=5, seq_len=6, variable_length=case == "ragged",
               stateful=case == "stateful")
    m = _model(cfg, dtype=torch.float64)
    B, T, V = 5, 6, 64
    x, y, *l = D.synthetic_next_token(B, T, V, seed=3, variable_length=case == "ragged")
    x, y = torch.as_tensor(x), torch.as_tensor(y)
    lengths = torch.as_tensor(l[0]) if case == "ragged" else None
    state = None
    if case == "stateful":
        g = torch.Generator().manual_seed(4)
        state = [(torch.randn(B, h, generator=g, dtype=torch.float64) * 0.5, torch.randn(B, h, generator=g, dtype=torch.float64) * 0.5)
                 for h in (16, 16)]
    emb, lstm, bias, perm = _torch_lm(m)
    loss, logits, _ok = m(x, y, lengths, state=state)
    loss.backward()
    want_loss, want_logits = _torch_forward(emb, lstm, bias, x, y, lengths, state)
    want_loss.backward()
    keep = ref.step_mask(lengths, B, T)
    assert torch.allclose(loss, want_loss, rtol=1e-12, atol=1e-12)
    assert torch.allclose(logits[keep], want_logits[keep], rtol=1e-12, atol=1e-12)
    # the table's gradient is the sum of both uses (the softmax's share alone is not it)
    assert torch.allclose(m.embedding.weights.grad, emb.weight.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(m.head.bias.grad, bias.grad, rtol=1e-12, atol=1e-12)
    for l, layer in enumerate(m.rnn.layers):
        for k, name in (("w_x", "weight_ih"), ("w_h", "weight_hh"), ("bias", "bias_ih")):
            got = perm(getattr(layer, k).grad)
            assert torch.allclose(got, getattr(lstm, f"{name}_l{l}").grad, rtol=1e-12, atol=1e-12), (l, k)


# ---- the class-major reference ops --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ragged", [False, True])
def test_reference_xent_class_major_is_the_transpose(ragged):
    g = torch.Generator().manual_seed(1)
    T, B, H, C = 5, 4, 8, 30
    h = torch.randn(T, B, H, generator=g, dtype=torch.float64)
    W = torch.randn(H, C, generator=g, dtype=torch.float64)
    b = torch.randn(C, generator=g, dtype=torch.float64)
    labels = torch.randint(0, C, (B, T), generator=g)
    lengths = torch.tensor([5, 1, 0, 3], dtype=torch.int32) if ragged else None
    a = ref.vocab_xent_per_step(h, W, b, labels, lengths)
    t = ref.vocab_xent_per_step(h, W.t().contiguous(), b, labels, lengths, class_major=True)
    assert all(torch.equal(u, v) for u, v in zip(a, t))
    from lstm_tensorspark_b200.ops import functional as F
    tab = W.t().contiguous().requires_grad_(True)
    F.vocab_xent_per_step(h, tab, b, labels, lengths, class_major=True)[0].backward()
    Wg = W.clone().requires_grad_(True)
    F.vocab_xent_per_step(h, Wg, b, labels, lengths)[0].backward()
    assert torch.allclose(tab.grad, Wg.grad.t(), rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("temperature", [0.0, 0.7])
def test_reference_sample_class_major_is_the_transpose(temperature):
    g = torch.Generator().manual_seed(2)
    B, H, C = 6, 8, 40
    h, W, b = torch.randn(B, H, generator=g), torch.randn(H, C, generator=g), torch.randn(C, generator=g)
    a = ref.vocab_sample(h, W, b, temperature, 11, 3, row0=2)
    t = ref.vocab_sample(h, W.t().contiguous(), b, temperature, 11, 3, row0=2, class_major=True)
    assert torch.equal(a[0], t[0]) and torch.equal(a[1], t[1])
    from lstm_tensorspark_b200.ops import functional as F
    assert torch.equal(F.vocab_sample(h, W.t().contiguous(), b, temperature, 11, 3, class_major=True)[0],
                       F.vocab_sample(h, W, b, temperature, 11, 3)[0])


def test_evaluation_logits_read_the_table():
    m = _model(_cfg(tie_embeddings=True))
    h = torch.randn(7, 16)
    assert torch.allclose(m.head_logits(h), h @ m.embedding.weights.t() + m.head.bias, rtol=1e-6, atol=1e-6)


# ---- checkpoints and runs -----------------------------------------------------------------------------------------------------
def _base(tmp_path, **kw):
    base = dict(hidden_units="32", in_features=32, seq_len=12, batch_size=32, vocab_size=64, next_token=True, synthetic=512,
                device="cpu", quiet=True, init="scaled", learning_rate=2e-2, steps_mode="epochs", evaluate_every=20,
                tie_embeddings=True, checkpoint_path=str(tmp_path / "ck"), output_path=str(tmp_path / "out"))
    base.update(kw)
    return base


def _last_checkpoint(tmp_path):
    from lstm_tensorspark_b200.utils import checkpoint as ckpt
    return ckpt.latest_checkpoint(ckpt.find_latest_run(str(tmp_path / "ck"), None))


def test_tied_checkpoints_resume_and_refuse_the_other_setting(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    from lstm_tensorspark_b200.utils import checkpoint as ckpt
    # a straight run of 2 epochs against 1 epoch + a resumed one: the same final weights, bit for bit
    straight = tmp_path / "straight"
    run_job(Config(epochs=2, **_base(straight, synthetic=64, evaluate_every=2)).validate(), standalone=True)
    run_job(Config(epochs=1, **_base(tmp_path, synthetic=64, evaluate_every=2)).validate(), standalone=True)
    variables, meta, _ = ckpt.load(_last_checkpoint(tmp_path))
    assert "Dense1/weights" not in variables and "Embedding/weights" in variables and "Dense1/bias" in variables
    assert ckpt.recorded_settings(meta)["tie_embeddings"] is True
    run_job(Config(epochs=2, use_pretrained_model=True, **_base(tmp_path, synthetic=64, evaluate_every=2)).validate(), standalone=True)
    a = ckpt.load(_last_checkpoint(straight))[0]
    b = ckpt.load(_last_checkpoint(tmp_path))[0]
    assert set(a) == set(b) and all(torch.equal(a[k], b[k]) for k in a)
    # eval / generate / resume without the flag: refused, the flag named
    untied = _base(tmp_path, synthetic=64, tie_embeddings=False)
    for mode in ("eval", "generate"):
        with pytest.raises(ValueError, match="with --tie_embeddings.*add --tie_embeddings"):
            run_job(Config(mode=mode, **untied).validate(), standalone=True)
    with pytest.raises(ValueError, match="--tie_embeddings"):
        run_job(Config(epochs=3, use_pretrained_model=True, **untied).validate(), standalone=True)


def test_untied_checkpoint_is_refused_by_a_tied_run(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    run_job(Config(epochs=1, max_steps=2, **_base(tmp_path, synthetic=64, tie_embeddings=False)).validate(), standalone=True)
    for mode in ("eval", "generate"):
        with pytest.raises(ValueError, match="without --tie_embeddings.*drop --tie_embeddings"):
            run_job(Config(mode=mode, **_base(tmp_path, synthetic=64)).validate(), standalone=True)


def test_files_that_record_nothing_load_as_untied():
    m, t = _model(_cfg()), _model(_cfg(tie_embeddings=True))
    vu, vt = dict(m.named_reference_variables()), dict(t.named_reference_variables())
    m.check_compatible(vu, {"next_token": True, "vocab_size": 64})                # nothing recorded, Dense1/weights present
    with pytest.raises(ValueError, match="without --tie_embeddings"):
        t.check_compatible(vu, {"next_token": True, "vocab_size": 64})
    with pytest.raises(ValueError, match="--tie_embeddings"):                    # nothing recorded, no Dense1/weights
        m.check_compatible(vt, {"next_token": True, "vocab_size": 64})
    with pytest.raises(ValueError, match="--tie_embeddings"):                    # recorded tied, yet a Dense1/weights matrix
        t.check_compatible(vu, {"next_token": True, "vocab_size": 64, "tie_embeddings": True})
    t.check_compatible(vt, {"next_token": True, "vocab_size": 64, "tie_embeddings": True})


def test_averaged_model_records_the_flag(tmp_path):
    from lstm_tensorspark_b200.trainer import run_job
    base = _base(tmp_path, partitions=2, max_workers=1, epochs=1, max_steps=2, synthetic=128)
    run_job(Config(**base).validate(), standalone=False)
    blob = torch.load(os.path.join(base["output_path"], "averaged_model.pt"), weights_only=False)
    assert blob["meta"]["tie_embeddings"] is True and "Dense1/weights" not in blob["variables"]
    assert json.load(open(os.path.join(base["output_path"], "averaged_model.json")))["tie_embeddings"] is True
    assert "perplexity" in run_job(Config(mode="eval", **dict(base, partitions=1)).validate(), standalone=False)
    with pytest.raises(ValueError, match="add --tie_embeddings"):
        run_job(Config(mode="eval", **dict(base, partitions=1, tie_embeddings=False)).validate(), standalone=False)


def test_cli_trains_scores_and_generates(tmp_path):
    """``lstm-no-spark.py --next_token --tie_embeddings`` lowers the loss; the model it leaves is scored and continues prompts."""
    args = ["--synthetic", "512", "--next_token", "--tie_embeddings", "--vocab_size", "64", "--in_features", "32",
            "--hidden_units", "32", "--seq_len", "12", "--batch_size", "32", "--device", "cpu", "--init", "scaled",
            "--learning_rate", "0.02", "--steps_mode", "epochs", "--evaluate_every", "20",
            "--checkpoint_path", str(tmp_path / "ck"), "--output_path", str(tmp_path / "out")]
    env = dict(os.environ, PYTHONPATH=ROOT)
    log = tmp_path / "log.jsonl"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "lstm-no-spark.py"), "--epochs", "25", "--quiet", "--json_log", str(log)]
                       + args, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    rows = [json.loads(s) for s in open(log) if "perplexity" in s]
    assert rows[0]["perplexity"] > 2 * rows[-1]["perplexity"] and rows[-1]["perplexity"] < 8
    from lstm_tensorspark_b200.trainer import run_job
    ev = run_job(Config(mode="eval", **_base(tmp_path)).validate(), standalone=True)
    assert ev["perplexity"] < 8
    out = run_job(Config(mode="generate", **_base(tmp_path, synthetic=40, temperature=0.0, max_new_tokens=6)).validate(),
                  standalone=True)
    assert out["tokens"] == 240 and out["legal_fraction"] >= 0.8                    # chance: 4/64


# ---- two ranks ----------------------------------------------------------------------------------------------------------------
def _sync_check(rank, world):
    import torch.distributed as dist
    from lstm_tensorspark_b200.engine import TrainEngine
    from lstm_tensorspark_b200.parallel.comm import make_communicator
    dev = torch.device("cpu")
    comm = make_communicator("gloo", rank, world, dev, 60)
    cfg = Config(hidden_units="8,8", in_features=8, batch_size=6, seq_len=5, sync_mode="grad_allreduce", device="cpu",
                 learn_initial_state=False, init="scaled", partitions=world, variable_length=True, vocab_size=16, next_token=True,
                 tie_embeddings=True, average_scope="all")
    eng = TrainEngine(cfg, rank, world, comm, batch_size=6, device=dev, dtype=torch.float32)
    H, V = 8, 16
    no_w = all(tuple(p.shape) != (H, V) for p in eng.flat.params) and eng.model.head.weights is None
    x, y, l = (torch.as_tensor(a) for a in D.synthetic_next_token(6, 5, 16, seed=rank, variable_length=True))
    for _ in range(4):
        eng.step(x, y, l)
    all_w = [torch.zeros_like(eng.flat.data) for _ in range(world)]
    dist.all_gather(all_w, eng.flat.data)
    comm.close()
    return no_w and all(torch.equal(all_w[0], w) for w in all_w)


def test_two_ranks_grad_allreduce_stay_equal():
    from lstm_tensorspark_b200.parallel.launch import launch
    assert all(launch(_sync_check, 2, args=()))
