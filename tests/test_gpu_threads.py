"""GPU: contexts driven from several host threads at once, every output bit for bit against the oracle.

One context must not be used concurrently, but distinct contexts may run at the same time from different threads
(include/prime_stereo_b200.h, Threading), and the bindings release the GIL in every call, so they really do overlap.

- The shared-memory limit race, made deterministic: a kernel's dynamic shared-memory limit is one value per device for
  the whole process, so a context that lowered it between another thread's set and launch would fail that launch.  The
  interposer tests/gate/libsmem_gate.so holds thread A right after its set until thread B sets the same kernel's limit or
  a second passes; tests/gate/race.py runs the pair in a fresh process (the limits start unset) under LD_PRELOAD.  Each
  case needs the gate to have held once, so it cannot pass without having opened the window.
- Free-running: the whole pairwise sweep (tests/config_sweep.py) on one thread per context at once, plus four contexts
  whose streaming-filter launches differ in shared memory; TorchStereo contexts on their own threads and torch streams;
  one context handed from thread to thread; per-thread creation errors; a multi-device context on devices [0, 0] beside a
  plain one.  Each runs a fixed number of frames, once."""
import ctypes as C
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import config_sweep as S
import test_gpu_config_sweep as SW
from oracle import oracle as O
from primestereomatch_b200 import DispEst, capi, synth
from test_gpu_config_sweep import mismatches, report, run_step

torch = pytest.importorskip("torch")

from primestereomatch_b200 import TorchStereo  # noqa: E402

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GATE = os.path.join(HERE, "gate", "libsmem_gate.so")
RACE = os.path.join(HERE, "gate", "race.py")
W, H = 140, 48
JOIN_S = 600   # no thread here should take more than a few seconds; a join past this is a hang, reported as one


def pair(seed, D=48):
    """a u8 stereo pair of W x H with noise on the right view"""
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=seed)
    rng = np.random.default_rng(seed)
    return l8, np.clip(r8.astype(np.int16) + rng.integers(-12, 13, r8.shape), 0, 255).astype(np.uint8)


def oracle_frame(l8, r8, D, window=8, eps=1e-4, fgf=None):
    """the raw and filtered volumes and both maps of [0, D) as a context with these settings computes them"""
    l, r = O.u8_to_f32(l8), O.u8_to_f32(r8)
    _, _, lraw, rraw = O.cost_const(l, r, D)
    if fgf:
        lf, rf = O.cost_filter_fgf(l, r, lraw, rraw, fgf, window=window, eps=eps)
    else:
        lf, rf = O.cost_filter(l, r, lraw, rraw, window=window, eps=eps)
    return {"lraw": lraw, "rraw": rraw, "lvol": lf, "rvol": rf, "lmap": O.wta(lf), "rmap": O.wta(rf)}


def diff(got, want, what):
    """-> [] or one line saying where got differs from want"""
    if got.shape != want.shape or got.dtype != want.dtype:
        return [f"{what}: {got.dtype} {got.shape} vs {want.dtype} {want.shape}"]
    if np.array_equal(got, want):
        return []
    bad = np.argwhere(got != want)
    i = tuple(bad[0])
    return [f"{what}: {len(bad)} of {got.size} differ, first at {list(i)}: {got[i]!r} vs {want[i]!r}"]


def run_threads(targets):
    """start one thread per callable, join them all -> the callables' exceptions as text (a thread still alive after
    JOIN_S counts as one)"""
    errors = []

    def wrap(f):
        def go():
            try:
                f()
            except BaseException as e:   # noqa: BLE001 -- reported after join
                errors.append(f"{type(e).__name__}: {e}")
        return go

    threads = [threading.Thread(target=wrap(f)) for f in targets]
    for t in threads:
        t.start()
    for t in threads:
        t.join(JOIN_S)
        if t.is_alive():
            errors.append(f"{t.name} still running after {JOIN_S} s")
    return errors


# ---- the limit race, held open by the gate -------------------------------------------------------------------------------
def ctx(D, window=None, eps=1e-4, fgf=None, volumes=True, **kwargs):
    return {"D": D, "kwargs": kwargs, "window": window, "eps": eps, "fgf": fgf, "volumes": volumes}


# (name, context A, context B, bytes A's launch asks for).  Thread A runs the larger launch.  The sizes are the launchers'
# own at W x H = 140 x 48: the streaming filter takes 512 bytes per thread, 128 threads at a slice count that is a multiple
# of 4 but not of 3 and 96 otherwise (65536 / 49152); the window filter win_smem_bytes(K, min(W, 258 - 2K) + K - 1)
# (91312 at window 16 / 62976 at window 5); the Fast Guided Filter fgf_smem_bytes(2 (window / rate) + 1) (107904 at rate
# 2 / 71744 at rate 4).
GATE_CASES = [
    ("stream_d64_d63", ctx(64), ctx(63), 65536),
    ("stream_blocked_d100_d63", ctx(100, block_slices=64, volumes=False), ctx(63), 65536),
    ("window16_window5", ctx(48, window=16), ctx(48, window=5, eps=1e-3), 91312),
    ("fgf2_fgf4", ctx(48, fgf=2), ctx(48, fgf=4), 107904),
]


@pytest.mark.parametrize("name,a,b,min_bytes", GATE_CASES, ids=[c[0] for c in GATE_CASES])
def test_limit_held_open_between_set_and_launch(name, a, b, min_bytes, tmp_path):
    assert os.path.exists(GATE), f"{GATE} is missing: __graft_entry__.build() makes it"
    frames = {}
    for i, v in enumerate("ab"):
        frames["l" + v], frames["r" + v] = pair(71 + i)
    np.savez(tmp_path / "frames.npz", **frames)
    spec = {"gate": GATE, "min_bytes": min_bytes, "timeout_ms": 1000, "frames": str(tmp_path / "frames.npz"),
            "out": str(tmp_path / "out.npz"), "a": a, "b": b}
    (tmp_path / "spec.json").write_text(json.dumps(spec))
    env = dict(os.environ, LD_PRELOAD=GATE)
    p = subprocess.run([sys.executable, RACE, str(tmp_path / "spec.json")], env=env, capture_output=True, text=True,
                       timeout=300)
    assert p.returncode == 0, f"driver exited with {p.returncode}:\n{p.stderr[-4000:]}"
    res = json.loads(p.stdout.strip().splitlines()[-1])
    print(f"{name}: gate {res['gate']}")
    assert res["forwards"] == 1, "the gate found no CUDA runtime to forward to"
    assert res["held"] and res["gate"]["holds"] >= 1, \
        f"the gate never held a set of >= {min_bytes} bytes, so the window was not opened: {res}"
    errs = {k: v for k, v in res["errors"].items() if v is not None}
    assert not errs, f"frames failed with the other thread's set inside the window (gate {res['gate']}): {errs}"
    out = np.load(tmp_path / "out.npz")
    lines = []
    for v, spec_v in (("a", a), ("b", b)):
        want = oracle_frame(frames["l" + v], frames["r" + v], spec_v["D"], spec_v["window"] or 8, spec_v["eps"],
                            spec_v["fgf"])
        keys = ("lraw", "rraw", "lvol", "rvol", "lmap", "rmap") if spec_v["volumes"] else ("lmap", "rmap")
        for k in keys:
            lines += diff(out[f"{v}_{k}"], want[k], f"context {v.upper()} {k}")
    assert not lines, "\n".join(lines)


# ---- the whole sweep at once ---------------------------------------------------------------------------------------------
# Four more contexts whose streaming-filter launches differ in shared memory (the sweep's D = 48, 300 and blocks of 7 and
# 5 all run 96 threads): D = 64 and the range [4, 68) at 128 threads, D = 63 at 96, D = 100 in 64-slice blocks at both.
EXTRA_FORMATS = {"u8_d64": (64, None), "u8_d63": (63, None), "u8_d68": (68, None), "u8_d100": (100, None)}
EXTRA_KINDS = {"range4": {"min_disp": 4}, "blocked64": {"block_slices": 64}}
EXTRA_GROUPS = [("unblocked", "u8_d64"), ("unblocked", "u8_d63"), ("range4", "u8_d68"), ("blocked64", "u8_d100")]
EXTRA_STEPS = [{"filter": "exact", "outputs": "none"}, {"filter": "mixed", "outputs": "costs"},
               {"filter": "exact", "outputs": "runner_up", "views": "left"}]


@pytest.fixture
def sweep_with_extras(monkeypatch):
    """the sweep's configurations and the four extra contexts' (groups after the sweep's), their levels registered with
    config_sweep for the duration of the test"""
    for k, v in EXTRA_FORMATS.items():
        monkeypatch.setitem(S.FORMATS, k, v)
    for k, v in EXTRA_KINDS.items():
        monkeypatch.setitem(S.KINDS, k, v)
    configs = list(SW.CONFIGS)
    for i, (kind, fmt) in enumerate(EXTRA_GROUPS):
        gi = len(SW.GROUPS) + i
        for si, step in enumerate(EXTRA_STEPS):
            c = {**S.DEFAULT, "kind": kind, "format": fmt, **step, "group": gi, "step": si}
            monkeypatch.setitem(SW.INDEX, (gi, si), len(configs))
            configs.append(c)
    return configs


def test_whole_sweep_on_concurrent_contexts(sweep_with_extras):
    configs = sweep_with_extras
    seqs = {}
    for c in configs:
        seqs.setdefault(c["group"], []).append(c)
    # every step's frames and expected outputs first, so that the device calls of the threads overlap
    frames = {id(c): S.frames(c, S.step_seed(c)) for c in configs}
    want = {id(c): S.expect(c, frames[id(c)]) for c in configs}
    rounds = max(len(s) for s in seqs.values())
    barrier = threading.Barrier(len(seqs), timeout=JOIN_S)
    failures = {gi: [] for gi in seqs}

    def worker(seq):
        def go():
            out = failures[seq[0]["group"]]
            W_, H_, D, bits = S.geometry(seq[0])
            blank = np.zeros((H_, W_, 3), np.uint8)
            de = None
            try:
                de = DispEst(blank, blank, D, map_bits=bits, **S.KINDS[seq[0]["kind"]])
            except capi.PsmError as e:
                out.append((SW.INDEX[seq[0]["group"], 0], seq[0], None, [f"creation raised {e}"]))
            prev = None
            for rnd in range(rounds):
                barrier.wait()   # steps advance in rounds; a thread whose sequence is done still waits
                if de is None or rnd >= len(seq):
                    continue
                c = seq[rnd]
                try:
                    lines = mismatches(run_step(de, prev, c, frames[id(c)]), want[id(c)])
                except Exception as e:   # noqa: BLE001 -- any failure is this step's; the thread goes on to the barrier
                    lines = [f"raised {type(e).__name__}: {e}"]
                if lines:
                    out.append((SW.INDEX[c["group"], c["step"]], c, prev, lines))
                prev = c
            if de is not None:
                de.close()
        return go

    errors = run_threads([worker(s) for s in seqs.values()])
    assert not errors, "\n".join(errors)
    bad = [f for gi in sorted(failures) for f in failures[gi]]
    if bad:
        pytest.fail(f"{len(bad)} of {len(configs)} configurations failed with {len(seqs)} contexts running at once; each "
                    "is run again below on a fresh context on one thread:\n" + report(bad), pytrace=False)


# ---- TorchStereo on several threads, each on its own stream -------------------------------------------------------------
TORCH_CONTEXTS = [   # (D, guided-filter window and eps or None, FGF rate or None)
    (64, None, None), (63, None, None), (48, (5, 1e-3), None), (48, None, 2), (48, (16, 1e-4), None), (48, None, 4),
]
TORCH_FRAMES = 6


def test_torch_stereo_threads_with_own_streams():
    scenes = [pair(101), pair(102)]
    want = {}
    for i, (D, gf, fgf) in enumerate(TORCH_CONTEXTS):
        window, eps = gf or (8, 1e-4)
        for s, (l8, r8) in enumerate(scenes):
            o = oracle_frame(l8, r8, D, window, eps, fgf)
            want[i, s] = (o["lmap"], o["rmap"])
    got = {}

    def worker(i):
        D, gf, fgf = TORCH_CONTEXTS[i]

        def go():
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream), TorchStereo(W, H, D, device=0) as ts:
                if gf:
                    ts.setGuidedFilter(*gf)
                if fgf:
                    ts.setSubsampleRate(fgf)
                dev = [tuple(torch.from_numpy(x).cuda() for x in sc) for sc in scenes]
                maps = [ts.match(*dev[f % 2], fgf=fgf is not None) for f in range(TORCH_FRAMES)]
                stream.synchronize()
                got[i] = [(lm.cpu().numpy(), rm.cpu().numpy()) for lm, rm in maps]
        return go

    errors = run_threads([worker(i) for i in range(len(TORCH_CONTEXTS))])
    assert not errors, "\n".join(errors)
    lines = []
    for i, ctx_maps in got.items():
        for f, (lm, rm) in enumerate(ctx_maps):
            wl, wr = want[i, f % 2]
            lines += diff(lm, wl, f"context {TORCH_CONTEXTS[i]} frame {f} left") + \
                diff(rm, wr, f"context {TORCH_CONTEXTS[i]} frame {f} right")
    assert not lines, "\n".join(lines)


# ---- one context handed between threads ----------------------------------------------------------------------------------
def test_context_handed_between_threads():
    """created on one thread, frames on a second and a third in turn, destroyed on a fourth"""
    D = 48
    scenes = [pair(201), pair(202)]
    want = [oracle_frame(l8, r8, D) for l8, r8 in scenes]
    box, lines = {}, []

    def create():
        box["de"] = DispEst(*scenes[0], D)

    def frames(first):
        def go():
            de = box["de"]
            for f in range(first, first + 2):
                s = f % 2
                de.setInputImages(*scenes[s])
                de.CostConst_GPU()
                de.CostFilter_GPU()
                lines.extend(diff(de.read_cost_volume(0), want[s]["lvol"], f"frame {f} left volume"))
                de.DispSelect_GPU()
                lines.extend(diff(de.lDisMap, want[s]["lmap"], f"frame {f} left map") +
                             diff(de.rDisMap, want[s]["rmap"], f"frame {f} right map"))
        return go

    def destroy():
        box["de"].close()

    steps = (("create", create), ("frames 0-1", frames(0)), ("frames 2-3", frames(2)), ("destroy", destroy))
    for name, step in steps:   # one thread after another: the context is never shared
        errors = run_threads([step])
        assert not errors, f"{name}: " + "\n".join(errors)
    assert not lines, "\n".join(lines)


# ---- per-thread creation errors -----------------------------------------------------------------------------------------
def test_creation_errors_are_per_thread():
    """two threads fail psm_create for different reasons at the same moment; each reads its own text from
    psm_last_error(NULL), and a third thread that never failed reads an empty string"""
    L = capi.lib()
    barrier = threading.Barrier(3, timeout=JOIN_S)
    results = {}
    cases = {"geometry": (0, H, 64, 0), "device": (W, H, 64, 9999), "none": None}

    def worker(name):
        def go():
            barrier.wait()
            rc = None
            if cases[name] is not None:
                ctx = C.c_void_p()
                rc = L.psm_create(C.byref(ctx), *cases[name])
                if rc == capi.PSM_OK:
                    L.psm_destroy(ctx)
            barrier.wait()   # both failures are in before anyone reads
            results[name] = (rc, L.psm_last_error(None).decode())
        return go

    errors = run_threads([worker(n) for n in cases])
    assert not errors, "\n".join(errors)
    (grc, gtext), (drc, dtext), (_, ntext) = results["geometry"], results["device"], results["none"]
    assert grc == capi.PSM_EINVAL and "bad geometry W=0" in gtext, results
    assert drc == capi.PSM_ECUDA and "CUDA device 9999 not available" in dtext, results
    assert ntext == "", results


# ---- co-located shards beside a plain context ---------------------------------------------------------------------------
def test_multi_device_shards_beside_plain_context():
    """a context of two shards on device 0 (D = 63: 31 and 32 slices, whose streaming-filter launches differ in shared
    memory) on one thread, a plain D = 64 context on another"""
    scenes = [pair(301), pair(302)]
    setups = {"multi": (63, {"devices": [0, 0]}), "plain": (64, {})}
    want = {(k, s): oracle_frame(*scenes[s], D) for k, (D, _) in setups.items() for s in range(2)}
    lines = []

    def worker(k):
        D, kwargs = setups[k]

        def go():
            with DispEst(*scenes[0], D, **kwargs) as de:
                for f in range(4):
                    s = f % 2
                    de.setInputImages(*scenes[s])
                    de.CostConst_GPU()
                    de.CostFilter_GPU()
                    de.DispSelect_GPU()
                    lines.extend(diff(de.lDisMap, want[k, s]["lmap"], f"{k} frame {f} left map") +
                                 diff(de.rDisMap, want[k, s]["rmap"], f"{k} frame {f} right map"))
        return go

    errors = run_threads([worker(k) for k in setups])
    assert not errors, "\n".join(errors)
    assert not lines, "\n".join(lines)
