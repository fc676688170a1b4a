"""CPU checks of R2D2: its built-in configs, the value rescaling pair h / h^-1, the loss's closed-form gradient (the one
jb_r2d2_loss writes) against float64 autograd, the oracle's LSTM against torch.nn.LSTM with episode resets, the
SequenceAssembler's windows across episode ends, and the frame-ring sizing the agent uses."""
import numpy as np
import pytest
import torch

from oracle import r2d2 as orr


def test_r2d2_configs():
    from jorldy_b200 import config as cfg
    paths = sorted(p for p in cfg.available() if p.split(".")[1] == "r2d2")
    assert paths == [f"config.r2d2.{e}" for e in ("atari", "cartpole", "mountaincar")]
    atari = cfg.load("config.r2d2.atari").agent
    want = dict(name="r2d2", network="r2d2", head="cnn", gamma=0.997, n_step=5, seq_len=80, n_burn_in=40, batch_size=64,
                buffer_size=100000, target_update_period=2500, alpha=0.9, beta=0.6, eta=0.9, hidden_size=512,
                clip_grad_norm=40.0)
    assert {k: atari[k] for k in want} == want
    assert cfg.load("config.r2d2.atari").optim == dict(name="adam", lr=1e-4, eps=1e-3)
    assert "distributed_batch_size" not in cfg.load("config.r2d2.atari").train      # the batch stays 64 sequences
    for env in ("cartpole", "mountaincar"):
        c, ref = cfg.load(f"config.r2d2.{env}"), cfg.load(f"config.ape_x.{env}")
        assert c.agent == dict(ref.agent, name="r2d2", network="r2d2", seq_len=16, n_burn_in=8, n_step=4, eta=0.9,
                               zero_padding=True)
        assert c.env == ref.env and c.optim == ref.optim and c.train == ref.train


def test_value_rescaling_round_trip():
    x = torch.cat([torch.linspace(0.0, 1.0, 1001), torch.logspace(0, 4, 2001)]).to(torch.float64)
    x = torch.cat([x, -x])
    for v in (x, orr.value_h_inv(x)):
        back = orr.value_h(orr.value_h_inv(v)) if v is x else orr.value_h_inv(orr.value_h(v))
        assert (back - v).abs().max().item() <= 1e-12 * max(1.0, v.abs().max().item())
    assert orr.value_h(torch.tensor(0.0, dtype=torch.float64)).item() == 0.0


@pytest.mark.parametrize("n", [1, 3])
def test_loss_closed_form_gradient_matches_autograd(n):
    rs = np.random.RandomState(n)
    B, T, A, gamma, eta, alpha = 5, 7, 4, 0.997, 0.9, 0.9
    t = lambda *s: torch.from_numpy(rs.standard_normal(s))
    q = t(B, T, A).requires_grad_(True)
    qn, qt = t(B, T, A), 10 * t(B, T, A)
    act = torch.from_numpy(rs.randint(A, size=(B, T)))
    rew, done = t(B, T + n), torch.from_numpy((rs.uniform(size=(B, T + n)) < 0.2).astype(np.float64))
    w = torch.from_numpy(rs.uniform(0.1, 1.0, size=B))
    L, td, prio = orr.loss(q, qn, qt, act, rew, done, w, gamma, n, eta, alpha)
    L.backward()
    closed = torch.zeros(B, T, A, dtype=torch.float64)
    closed.scatter_(-1, act.unsqueeze(-1), (-2.0 * w.unsqueeze(-1) * td.detach() / (B * T)).unsqueeze(-1))
    assert torch.allclose(q.grad, closed, rtol=1e-12, atol=1e-15)
    # the target: explicit loops
    for b in range(B):
        for s in range(T):
            a_star = int(qn[b, s].argmax())
            y = float(orr.value_h_inv(qt[b, s, a_star]))
            for i in range(n - 1, -1, -1):
                y = float(rew[b, s + i]) + (1.0 - float(done[b, s + i])) * gamma * y
            y = float(orr.value_h(torch.tensor(y, dtype=torch.float64)))
            assert abs(float(td[b, s]) - (y - float(q.detach()[b, s, act[b, s]]))) < 1e-9
        a = td[b].detach().abs()
        assert abs(float(prio[b]) - (eta * float(a.max()) + (1 - eta) * float(a.mean())) ** alpha) < 1e-12


@pytest.mark.parametrize("reset_kind", ["none", "all", "random"])
def test_oracle_lstm_matches_torch_lstm_with_resets(reset_kind):
    rs = np.random.RandomState(0)
    S, B, Z, H = 9, 4, 6, 5
    ref = torch.nn.LSTM(Z, H).to(torch.float64)
    p = {f"lstm.{k}": v.detach() for k, v in ref.state_dict().items()}
    z = torch.from_numpy(rs.standard_normal((S, B, Z)))
    reset = np.zeros((S, B))
    if reset_kind == "all":
        reset[:] = 1
    elif reset_kind == "random":
        reset = (rs.uniform(size=(S, B)) < 0.3).astype(np.float64)
    h0, c0 = torch.from_numpy(rs.standard_normal((B, H))), torch.from_numpy(rs.standard_normal((B, H)))
    hs, (h, c) = orr.lstm(p, z, torch.from_numpy(reset), h0, c0)
    for b in range(B):      # torch.nn.LSTM run segment by segment, restarting from zeros at every reset
        hb, cb = h0[b:b + 1].unsqueeze(0), c0[b:b + 1].unsqueeze(0)
        for s in range(S):
            if reset[s, b]:
                hb, cb = torch.zeros_like(hb), torch.zeros_like(cb)
            out, (hb, cb) = ref(z[s:s + 1, b:b + 1], (hb, cb))
            assert torch.allclose(hs[s, b], out[0, 0], rtol=0, atol=1e-13)
        assert torch.allclose(c[b], cb[0, 0], atol=1e-13)


def test_sequence_assembler_windows_across_episode_ends():
    from jorldy_b200.core.collect import SequenceAssembler
    Tb, T, n, N, H = 2, 4, 1, 3, 2
    asm = SequenceAssembler(Tb, T, n)
    L, P = asm.L, asm.period
    assert (L, P) == (7, 2)
    rs = np.random.RandomState(0)
    done = rs.uniform(size=(40, N)) < 0.25
    done[L - 1, 0] = done[L, 1] = True        # a done at a window's last step and just before a window's first step
    emitted, kept = [], []
    reset = np.ones(N)
    for t in range(40):
        tr = {"state": torch.full((N, 2), float(t)), "action": torch.full((N,), t, dtype=torch.int64),
              "prev_action": torch.full((N,), t - 1, dtype=torch.int64), "reset": torch.tensor(reset, dtype=torch.float32),
              "reward": torch.full((N,), float(t)), "done": torch.tensor(done[t], dtype=torch.float32)}
        if asm.starts_window():
            tr.update(h0=torch.full((N, H), float(t)), c0=torch.full((N, H), -float(t)))
        out = asm.push(tr)
        kept.append(len(asm.snap))
        if out is not None:
            emitted.append((t, out))
        reset = done[t].astype(np.float64)
    assert [t for t, _ in emitted] == list(range(L - 1, 40, P))
    assert max(kept) <= -(-L // P) + 1
    for t, out in emitted:
        start = t - L + 1
        steps = np.arange(start, t + 1)
        assert out["state"].shape == (N, L, 2) and out["h0"].shape == (N, H)
        assert np.array_equal(out["action"].numpy(), np.tile(steps, (N, 1)))
        assert np.array_equal(out["reward"].numpy(), np.tile(steps, (N, 1)).astype(np.float32))
        assert np.array_equal(out["done"].numpy().T, done[start:t + 1].astype(np.float32))
        want_reset = np.concatenate([np.ones((1, N)) if start == 0 else done[start - 1:start], done[start:t]]).T
        assert np.array_equal(out["reset"].numpy(), want_reset.astype(np.float32))
        assert torch.equal(out["h0"], torch.full((N, H), float(start))) and torch.equal(out["c0"], -out["h0"])


def _max_frame_reach(F, capacity, lanes, store_period, L, reset_every):
    """Host model of one lane: pushes one frame per step plus one per reset; the replay keeps the newest `capacity`
    sequences of all lanes (one per lane every store_period steps).  Returns True if every frame the oldest kept
    sequence references (its L stacks, 3 frames of history each) is still in the ring of F frames."""
    per_lane = -(-capacity // lanes)
    steps = per_lane * store_period + L + 5 * store_period
    pos, pushed = [], 1                       # frame position of each step's state stack (the newest frame)
    for t in range(steps):
        pos.append(pushed - 1)
        pushed += 1 + (1 if (t + 1) % reset_every == 0 else 0)
    starts = [s for s in range(0, steps - L + 1, store_period)][-per_lane:]
    oldest = starts[0]
    return pos[oldest] - 3 >= pushed - F


@pytest.mark.parametrize("capacity,lanes", [(1000, 8), (4096, 16), (100000, 128)])
def test_sequence_frame_ring_sizing(capacity, lanes):
    from jorldy_b200.core.buffer.frame_store import frames_per_lane
    P, L = 40, 125
    F = frames_per_lane(capacity * P, lanes, L)
    assert _max_frame_reach(F, capacity, lanes, P, L, reset_every=16)
    assert not _max_frame_reach(F - 4 - (-(-capacity // lanes)) * P // 16 - L, capacity, lanes, P, L, reset_every=16)
