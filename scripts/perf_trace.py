"""Intra-step timeline of the persistent PPO kernel: clock64 stamps of the last step (debug trace, JB_FUSED_SKIP=256).

    python scripts/perf_trace.py [--config cartpole|continuous] [--batch B] --ghz F

--config cartpole: D=4, A=2 discrete (bench ppo_cartpole, B=256); continuous: D=11, A=3 Gaussian (bench ppo_continuous,
B=512).  --ghz converts clock64 ticks to microseconds: pass the SM clock the card actually ran at
(`nvidia-smi --query-gpu=clocks.max.sm`), it is not read here."""
import argparse, ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ap = argparse.ArgumentParser()
ap.add_argument("--config", choices=("cartpole", "continuous"), default="cartpole")
ap.add_argument("--batch", type=int, default=None)
ap.add_argument("--ghz", type=float, required=True)
args = ap.parse_args()
os.environ["JB_FUSED_SKIP"] = "256"

import numpy as np, torch
from jorldy_b200.core import Agent, Env
from jorldy_b200.core.collect import RolloutCollector
from jorldy_b200._lib import C

if args.config == "cartpole":
    env_name, D, A, kw, B = "cartpole", 4, 2, {}, args.batch or 256
else:
    env_name, D, A, kw, B = "hopper", 11, 3, {"network": "continuous_policy_value"}, args.batch or 512
N, T = 4096, 32
env = Env(env_name, num_envs=N, seed=0)
agent = Agent("ppo", state_size=D, action_size=A, hidden_size=512, batch_size=B, n_step=T, n_epoch=1,
              optim_config={"name": "adam", "lr": 2.5e-4}, device="cuda", run_step=10**9, use_fused=True, **kw)
col = RolloutCollector(env, agent, use_cuda_graph=False); col.collect()
agent.learn_rollout(col.rollout); col.rollout.t = T
st = agent._st; fr = agent._fused[B]
n = N * T // B
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
agent._cursor.zero_(); e0.record(); fr.run(st, n); e1.record(); torch.cuda.synchronize()
print(f"{args.config} B={B}: {e0.elapsed_time(e1)/n*1000:.1f} us/step over {n} steps (traced)")
tr = np.zeros((256, 48), np.int64)
C.jb_ppo_fused_trace(tr.ctypes.data_as(ctypes.c_void_p))
names = {0: "step start", 1: "P1 h1 generated", 2: "P1 panel landed", 3: "P1 mma", 4: "P1 reduce", 5: "P1 end", 6: "bar1",
         7: "critic means done", 8: "P3 job0 start", 9: "P3 job1 start", 10: "P3 job2 start", 11: "P3 job3+ start",
         12: "JB staged", 13: "JB dh2 gen", 14: "JB mma", 15: "JB reduce", 16: "JB end",
         17: "JA staged", 18: "JA dh2 gen", 19: "JA mma(last)", 20: "JA reduce(last)", 21: "JA end",
         22: "P3 jobs end", 28: "P1 stash issued", 29: "P1 stash landed",
         33: "JB dW1 staged", 34: "JB dW1 stored", 35: "P1 shuffles done", 36: "P1 ticket drawn",
         37: "row maths done (last arriver)", 38: "row table landed", 23: "norm partial + p/m/v issued", 24: "bar3", 25: "P5 fold", 26: "P5 end", 27: "bar5",
         39: "JC staged", 30: "JC end", 31: "JD counter reached", 32: "JD end"}
ghz = args.ghz
n = int((tr[:, 0] > 0).sum())               # CTAs of the launch
for cta in sorted({0, n // 2, n - 1}):
    t = tr[cta]
    print(f"--- CTA {cta}")
    order = sorted([i for i in names if t[i] > 0], key=lambda i: t[i])
    prev = t[0]
    for i in order:
        print(f"  {names[i]:28s} +{(t[i]-prev)/ghz/1000:6.2f} us   @{(t[i]-t[0])/ghz/1000:6.2f}")
        prev = t[i]
# barrier waits: arrival spread
for a_, b_, nm in [(5, 6, "bar1"), (23, 24, "bar3"), (26, 27, "bar5")]:
    arr = tr[:n, a_] - tr[:n, 0]; dep = tr[:n, b_] - tr[:n, 0]
    print(f"{nm}: arrive min {arr.min()/ghz/1000:.2f} max {arr.max()/ghz/1000:.2f} (cta {arr.argmax()}) | depart-arrive min {(dep - arr).min()/ghz/1000:.2f} us")
# P1 spans over all CTAs that ran a P1 tile.  A span ends at its slot and starts at the CTA's previous stamped slot of the
# chain; "row maths" is stamped only by a row tile's last arriver, so the span into bar1 arrival starts at the ticket for the
# others.  A CTA with several P1 tiles stamps slots 1..37 for its last tile (the earlier ones fall into "h1 generated").
# g_trace is not cleared between launches and clock64 is per SM, so a slot is used only if it lies inside this CTA's step.
chain = [(28, "stash issued"), (29, "stash landed"), (1, "h1 generated"), (2, "W2 panel landed"), (3, "mma"),
         (4, "reduce"), (35, "shuffles"), (36, "ticket"), (37, "row maths (last arrivers)"), (5, "bar1 arrival")]
us = lambda x: x / ghz / 1000
p1 = [c for c in range(n) if tr[c, 5] >= tr[c, 1] >= tr[c, 0] > 0]
spans = {s: [] for s, _ in chain}
at = {s: [] for s, _ in chain}
for c in p1:
    t = tr[c]; prev = t[0]
    for s, _ in chain:
        if t[s] < prev or t[s] > t[5]:
            continue
        spans[s].append(us(t[s] - prev)); at[s].append(us(t[s] - t[0])); prev = t[s]
print(f"P1 spans over {len(p1)} CTAs (us; span from the previous slot, @ from the step start)")
def table(rows):
    print(f"  {'span end':28s} {'CTAs':>4s} {'median':>7s} {'max':>7s}   {'@median':>7s} {'@max':>7s}")
    for nm, sp, a_ in rows:
        if sp:
            v, w = np.array(sp), np.array(a_)
            print(f"  {nm:28s} {len(v):4d} {np.median(v):7.2f} {v.max():7.2f}   {np.median(w):7.2f} {w.max():7.2f}")
table([(nm, spans[s], at[s]) for s, nm in chain])

# P3 spans over every CTA, per job kind.  The job map is round-robin (job = cta + i * CTAs) over nJB JB (dh1 tiles), nJA JA
# (pairs of dW2 tiles), nJC JC (head gradients) and nJD JD (dW1 folds) jobs; job i of a CTA stamps slot 8 + min(i, 3) at its
# start.  Each kind has one set of slots, so a CTA that runs two jobs of one kind keeps the stamps of the last one, and one
# whose job i >= 3 shares slot 11 with its other jobs i >= 3: such CTAs are counted only where the slots are unambiguous.
H = 512
MT, NTL = B // 32, H // 32
kinds = [("JB", MT * NTL), ("JA", NTL * ((NTL + 1) // 2)), ("JC", NTL), ("JD", NTL)]
first = np.cumsum([0] + [k[1] for k in kinds])
nJ3 = int(first[-1])
kind_of = lambda j: kinds[int(np.searchsorted(first, j, side="right")) - 1][0]
jobs = {c: list(range(c, nJ3, n)) for c in range(n)}
per_kind = {}
for c in range(n):
    for k, _ in kinds:
        idx = [i for i, j in enumerate(jobs[c]) if kind_of(j) == k]
        if idx:
            per_kind.setdefault(k, {})[c] = idx
shared = sorted({k for k, d in per_kind.items() for idx in d.values() if len(idx) > 1 or idx[-1] >= 3})
if shared:
    print(f"note: at B={B} some CTAs run several jobs of kind {', '.join(shared)} or a 4th+ job: "
          "their per-kind stamps belong to the last such job, its start slot is used only when unambiguous")
p3_chains = {"JB": [(12, "JB staged"), (13, "JB dh2 gen"), (14, "JB mma"), (15, "JB reduce"), (33, "JB dW1 partial"),
                    (34, "JB dW1 fold + store"), (16, "JB end")],
             "JA": [(17, "JA staged"), (18, "JA dh2 gen"), (19, "JA mma (last half)"), (20, "JA reduce (last half)"),
                    (21, "JA end")],
             "JC": [(39, "JC staged"), (30, "JC end")],
             "JD": [(31, "JD counter reached"), (32, "JD end")]}
inside = lambda t, s: t[0] < t[s] <= t[23]          # the slot was written during this CTA's traced step
print(f"P3 spans over {n} CTAs (us; span from the previous slot, @ from the step start)")
rows = []
for s, prev_s, nm in [(38, 6, "bar1 -> row table landed"), (7, 38, "critic means done")]:
    sp, a_ = [], []
    for c in range(n):
        t = tr[c]
        if inside(t, s) and inside(t, prev_s):
            sp.append(us(t[s] - t[prev_s])); a_.append(us(t[s] - t[0]))
    rows.append((nm, sp, a_))
table(rows)
for k, _ in kinds:
    rows = {s: ([], []) for s, _ in p3_chains[k]}
    for c, idx in per_kind.get(k, {}).items():
        t = tr[c]
        i = idx[-1]
        start = 8 + min(i, 3)
        prev = t[start] if (i < 3 or i == len(jobs[c]) - 1) and inside(t, start) else None
        for s, _ in p3_chains[k]:
            if not inside(t, s):
                continue
            if prev is not None and t[s] >= prev:
                rows[s][0].append(us(t[s] - prev)); rows[s][1].append(us(t[s] - t[0]))
            prev = t[s]
    print(f" {k} ({len(per_kind.get(k, {}))} CTAs)")
    table([(nm, *rows[s]) for s, nm in p3_chains[k]])
ends, arr = [], tr[:n, 23] - tr[:n, 0]
for c in range(n):
    if inside(tr[c], 22):
        ends.append(us(tr[c, 22] - tr[c, 0]))
print(f"  P3 jobs end @ median {np.median(ends):.2f} max {max(ends):.2f} us")
a_us = np.array([us(x) for x in arr])
q = np.percentile(a_us, [0, 10, 50, 90, 100])
print(f"bar3 arrival @ (us from step start) min {q[0]:.2f} p10 {q[1]:.2f} median {q[2]:.2f} p90 {q[3]:.2f} max {q[4]:.2f}")
desc = lambda c: "+".join(kind_of(j) for j in jobs[c]) or "none"
for c in np.argsort(-a_us)[:6]:
    print(f"  cta {c:3d} @ {a_us[c]:6.2f} us  jobs {desc(c)}")
by = {}
for c in range(n):
    by.setdefault(desc(c), []).append(a_us[c])
for d_, v in sorted(by.items()):
    print(f"  jobs {d_:16s} {len(v):4d} CTAs  bar3 arrival median {np.median(v):6.2f} max {max(v):6.2f} us")
