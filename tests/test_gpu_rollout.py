"""GPU tests of the device rollout storage (soundspaces_b200/rollout.py, ``ssb_rollout_*_batch``): every seeded script
of tests/rollout_models.py runs on the device once with patched copies of the stand-ins and once eagerly; storage,
returns, minibatches and torch's RNG must be bit-identical (to the eager run after every insert, and to the reference
golden), the advantages within 1e-5 of float64 and bit-identical across calls; inserts make no stream synchronisation
and each method one library launch; a memory row over capacity raises at ``compute_returns``; storage and arguments
that do not qualify run the originals."""
import os

import numpy as np
import pytest
import torch

import rollout_models as rm
from soundspaces_b200 import rollout as ro
from soundspaces_b200.renderer import WaveformOps

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "rollout_golden.npz")
DEV = torch.device("cuda", 0)
EAGER = dict(common=rm.CommonRolloutStorage, savi=rm.SaviRolloutStorage)
PATCHED = {k: ro.patch_rollout_storage(type("Patched" + v.__name__, (v,), {})) for k, v in EAGER.items()}
PATCHED_PPO = ro.patch_ppo(type("PatchedPPO", (rm.PPO,), {}))


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("host", [False, True])
@pytest.mark.parametrize("use_gae", [True, False])
@pytest.mark.parametrize("name", sorted(rm.SCRIPTS))
def test_patched_storage_is_bit_identical(golden, name, use_gae, host):
    """``host``: observations, rewards and masks on the CPU, as the stock AV-Nav / AV-WaN trainers pass them."""
    script = rm.SCRIPTS[name]
    eager_states, patched_states = [], []
    # SAVi's eager memory update needs its masks on the device (its trainer moves them there); the patched side
    # takes them from the host all the same
    eager = rm.run_script(script, EAGER, rm.PPO, use_gae, DEV, host and script["kind"] == "common",
                          on_insert=lambda st: eager_states.append(rm.state(st)))
    ctx = WaveformOps.get(DEV).ctx
    n0 = ctx.launch_count
    patched = rm.run_script(script, PATCHED, PATCHED_PPO, use_gae, DEV, host,
                            on_insert=lambda st: patched_states.append(rm.state(st)))
    # one launch per insert, compute_returns, minibatch and after_update: nothing fell back to the original
    per_rollout = script["S"] + 1 + sum(rm.MINI_BATCHES) + 1
    assert ctx.launch_count - n0 == script["rollouts"] * per_rollout
    assert len(eager_states) == len(patched_states) == script["rollouts"] * script["S"]
    for i, (e, p) in enumerate(zip(eager_states, patched_states)):
        assert e.keys() == p.keys()
        for k in e:
            assert _same(e[k], p[k]), f"insert {i}: {k}"
    prefix = rm.golden_key(name, use_gae)
    assert eager.keys() == patched.keys()
    for k in patched:
        if k.endswith("/adv"):          # the normalised advantages (and their minibatches): another summation order
            continue
        assert _same(patched[k], golden[f"{prefix}/{k}"]) and _same(patched[k], eager[k]), k
    S, N = script["S"], script["N"]
    for r in range(script["rollouts"]):
        adv = patched[f"{r}/adv"]
        ref = rm.advantages64(patched[f"{r}/returns"], patched[f"{r}/value_preds"])
        assert np.abs(adv - ref).max() < 1e-5
        for m, seed in zip(rm.MINI_BATCHES, rm.GENERATOR_SEEDS):   # the advantages' own minibatch gather
            torch.manual_seed(seed)
            perm = torch.randperm(N).numpy()
            nb = N // m
            want = np.stack([adv[:, perm[i * nb:(i + 1) * nb]].reshape(S * nb, 1) for i in range(m)])
            assert _same(patched[f"{r}/mb{m}/adv"], want), (r, m)


def _filled(name="savi", cls=None):
    """A storage of ``name`` filled with one rollout, and its next value."""
    script = rm.SCRIPTS[name]
    st = rm.make_storage(script, cls or PATCHED, DEV)
    g = np.random.default_rng(7)
    for _ in range(script["S"]):
        st.insert(*rm.to_device(rm.step_inputs(script, g), DEV))
    return st, torch.from_numpy(g.standard_normal((script["N"], 1), dtype=np.float32)).to(DEV)


@pytest.mark.parametrize("name", ["common", "savi"])
def test_advantages_are_deterministic_and_shared(name):
    st, nv = _filled(name)
    st.compute_returns(nv, True, 0.99, 0.95)
    a = PATCHED_PPO().get_advantages(st).clone()
    st.compute_returns(nv, True, 0.99, 0.95)
    b = PATCHED_PPO().get_advantages(st)
    eager, _ = _filled(name, EAGER)
    eager.compute_returns(nv, True, 0.99, 0.95)
    c = PATCHED_PPO().get_advantages(eager)          # eager storage: the kernel's advantage-only path
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(a, c)
    ref = rm.advantages64(st.returns.cpu().numpy(), st.value_preds.cpu().numpy())
    assert np.abs(a.cpu().numpy() - ref).max() < 1e-5


@pytest.mark.parametrize("host", [False, True])
@pytest.mark.parametrize("name", ["common", "savi"])
def test_insert_makes_no_synchronisation_and_one_launch_per_method(name, host):
    """With ``host``, the inputs the stock AV-Nav / AV-WaN trainers pass: CPU observations, rewards and masks."""
    script = rm.SCRIPTS[name]
    st = rm.make_storage(script, PATCHED, DEV)
    g = np.random.default_rng(3)
    steps = [rm.to_device(rm.step_inputs(script, g), DEV, host) for _ in range(script["S"])]
    ctx = WaveformOps.get(DEV).ctx
    torch.cuda.synchronize()
    counts = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for args in steps:
            before = ctx.launch_count
            st.insert(*args)
            counts.append(ctx.launch_count - before)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert counts == [1] * script["S"]
    nv = torch.zeros((script["N"], 1), device=DEV)
    before = ctx.launch_count
    st.compute_returns(nv, True, 0.99, 0.95)
    adv = PATCHED_PPO().get_advantages(st)
    assert ctx.launch_count - before == 1
    for m in rm.MINI_BATCHES:
        before = ctx.launch_count
        n = sum(1 for _ in st.recurrent_generator(adv, m))
        assert n == m and ctx.launch_count - before == m
    before = ctx.launch_count
    st.after_update()
    assert ctx.launch_count - before == 1


def test_memory_over_capacity_raises_at_compute_returns():
    st, nv = _filled("savi")
    st.after_update()
    st.em.masks[2].fill_(1.0)                    # row 2 now holds every slot, more than the capacity
    script = rm.SCRIPTS["savi"]
    g = np.random.default_rng(9)
    st.insert(*rm.to_device(rm.step_inputs(script, g), DEV))
    with pytest.raises(AssertionError, match=r"env rows \[2\].*first at step 0"):
        st.compute_returns(nv, True, 0.99, 0.95)
    st.compute_returns(nv, True, 0.99, 0.95)     # the status word was cleared: no stale error


def test_external_memory_patch_matches_eager_and_raises():
    cls = ro.patch_external_memory(type("PatchedEM", (rm.ExternalMemory,), {}))
    N, total, cap, dim = 5, 9, 4, 3
    eager, patched = rm.ExternalMemory(N, total, cap, dim), cls(N, total, cap, dim)
    eager.to(DEV)
    patched.to(DEV)
    g = np.random.default_rng(11)
    ctx = WaveformOps.get(DEV).ctx
    for i in range(20):
        feats = torch.from_numpy(g.standard_normal((N, dim), dtype=np.float32)).to(DEV)
        masks = torch.from_numpy((g.random((N, 1)) > 0.2).astype(np.float32))
        masks = masks if i % 2 else masks.to(DEV)
        eager.insert(feats, masks.to(DEV))
        before = ctx.launch_count
        patched.insert(feats, masks)
        assert ctx.launch_count - before == 1
        assert eager.idx == patched.idx
        assert torch.equal(eager.memory, patched.memory) and torch.equal(eager.masks, patched.masks)
    patched.masks[1].fill_(1.0)
    idx = patched.idx
    with pytest.raises(AssertionError, match=r"env rows \[1\]"):
        patched.insert(torch.zeros((N, dim), device=DEV), torch.ones((N, 1), device=DEV))
    assert patched.idx == idx
    patched.masks.zero_()
    patched.insert(torch.zeros((N, dim), device=DEV), torch.ones((N, 1), device=DEV))   # cleared: no stale error
    assert patched.idx == (idx + 1) % total


def test_storage_and_arguments_that_do_not_qualify_run_the_originals():
    script = rm.SCRIPTS["common"]
    ctx = WaveformOps.get(DEV).ctx
    # storage: a non-contiguous rewards tensor
    eager, patched = rm.make_storage(script, EAGER, DEV), rm.make_storage(script, PATCHED, DEV)
    for st in (eager, patched):
        st.rewards = st.rewards.transpose(0, 1).contiguous().transpose(0, 1)
    assert ro.rollout_layout_error(patched) == "rewards is not contiguous"
    g1, g2 = np.random.default_rng(1), np.random.default_rng(1)
    before = ctx.launch_count
    for _ in range(script["S"]):
        eager.insert(*rm.to_device(rm.step_inputs(script, g1), DEV))
        patched.insert(*rm.to_device(rm.step_inputs(script, g2), DEV))
    nv = torch.ones((script["N"], 1), device=DEV)
    eager.compute_returns(nv, True, 0.99, 0.95)
    patched.compute_returns(nv, True, 0.99, 0.95)
    torch.manual_seed(0)
    eb = list(eager.recurrent_generator(rm.PPO().get_advantages(eager), 2))
    torch.manual_seed(0)
    pb = list(patched.recurrent_generator(PATCHED_PPO().get_advantages(patched), 2))
    eager.after_update()
    patched.after_update()
    assert ctx.launch_count - before == 1        # only get_advantages's advantage-only launch
    assert all(np.array_equal(rm.state(eager)[k], v) for k, v in rm.state(patched).items())
    assert len(eb) == len(pb) == 2
    for a, b in zip(eb, pb):
        for k, v in rm.batch_arrays(b).items():
            assert k == "adv" or np.array_equal(rm.batch_arrays(a)[k], v), k
    # arguments: float64 observations and a non-contiguous hidden state go through copy_
    eager, patched = rm.make_storage(script, EAGER, DEV), rm.make_storage(script, PATCHED, DEV)
    g = np.random.default_rng(2)
    args = rm.to_device(rm.step_inputs(script, g), DEV)
    args[0] = {k: v.double() for k, v in args[0].items()}
    args[1] = args[1].transpose(0, 1).contiguous().transpose(0, 1)
    before = ctx.launch_count
    eager.insert(*args)
    patched.insert(*args)
    assert ctx.launch_count == before and patched.step == eager.step == 1
    assert all(np.array_equal(rm.state(eager)[k], v) for k, v in rm.state(patched).items())


def test_a_sensor_already_in_its_slot_is_not_copied():
    """``batch_obs(out=...)`` renders into the slot itself; the insert then copies every other field only."""
    script = rm.SCRIPTS["common"]
    eager, patched = rm.make_storage(script, EAGER, DEV), rm.make_storage(script, PATCHED, DEV)
    g = np.random.default_rng(4)
    ctx = WaveformOps.get(DEV).ctx
    for _ in range(3):
        args = rm.to_device(rm.step_inputs(script, g), DEV)
        for st in (eager, patched):
            st.observations["depth"][st.step + 1].copy_(args[0]["depth"])
        eager.insert(*args)
        obs = dict(args[0], depth=patched.observations["depth"][patched.step + 1])
        before = ctx.launch_count
        patched.insert(obs, *args[1:])
        assert ctx.launch_count - before == 1
    assert all(np.array_equal(rm.state(eager)[k], v) for k, v in rm.state(patched).items())


def test_get_advantages_hands_out_each_result_once():
    st, nv = _filled("common")
    st.compute_returns(nv, True, 0.99, 0.95)
    a = PATCHED_PPO().get_advantages(st)
    ref = a.clone()
    a.fill_(7.0)                                 # a caller's in-place edit
    b = PATCHED_PPO().get_advantages(st)
    assert b is not a and torch.equal(b, ref)


def test_entries_refuse_bad_arguments_and_shapes():
    import ctypes as C
    from soundspaces_b200 import _lib
    ops = WaveformOps.get(DEV)
    lib, h, stream = ops.lib, ops.ctx.handle, ops._stream()
    buf = torch.zeros(1024, device=DEV)
    p = buf.data_ptr()
    n0 = ops.ctx.launch_count
    field = lambda **kw: ops._rollout_fields([(kw.get("src", p), p + 2048, kw.get("row", 16), 0, 0,  # noqa: E731
                                               kw.get("T", 1), kw.get("outer", 1), kw.get("host", 0))])
    E_INVALID, E_SHAPE = -1, -4
    assert lib.ssb_rollout_insert_batch(h, 0, field(), 1, None, stream) == E_INVALID
    assert lib.ssb_rollout_insert_batch(h, 70000, field(), 1, None, stream) == E_SHAPE
    assert lib.ssb_rollout_insert_batch(h, 4, field(), 33, None, stream) == E_INVALID
    assert lib.ssb_rollout_insert_batch(h, 4, field(host=2), 1, None, stream) == E_INVALID
    assert lib.ssb_rollout_insert_batch(h, 4, field(host=1, T=2), 1, None, stream) == E_INVALID
    assert lib.ssb_rollout_insert_batch(h, 4, field(src=None), 1, None, stream) == E_INVALID
    assert lib.ssb_rollout_insert_batch(h, 4, field(row=0), 1, None, stream) == E_SHAPE
    assert lib.ssb_rollout_insert_batch(h, 4, field(row=1 << 46), 1, None, stream) == E_SHAPE
    em = _lib.RolloutMemory(p, p, None, p, 8, 9, 0, 0, 0, 0)       # capacity above the slots
    assert lib.ssb_rollout_insert_batch(h, 4, field(), 1, C.byref(em), stream) == E_INVALID
    em = _lib.RolloutMemory(p, p, None, p, 20000, 5, 0, 0, 0, 0)   # more slots than the kernel takes
    assert lib.ssb_rollout_insert_batch(h, 4, field(), 1, C.byref(em), stream) == E_SHAPE
    ret = lambda N, S, T, scan=1, adv=None: lib.ssb_rollout_returns_batch(  # noqa: E731
        h, N, S, T, scan, 1, 0.99, 0.94, p, p, p, p, p, adv, 1, stream)
    assert ret(0, 4, 4) == E_INVALID and ret(4, 4, 5) == E_INVALID and ret(4, 4, 4, scan=0) == E_INVALID
    assert ret(70000, 4, 4) == E_SHAPE and ret(4, 5000, 4) == E_SHAPE
    cols = (C.c_int64 * 300)(*range(300))
    assert lib.ssb_rollout_gather_batch(h, field(), 0, 4, None, 0, stream) == E_INVALID
    assert lib.ssb_rollout_gather_batch(h, field(), 1, 300, cols, 300, stream) == E_SHAPE
    assert lib.ssb_rollout_gather_batch(h, field(), 1, 2, cols, 1, stream) == E_INVALID   # column 1 >= max_col
    assert lib.ssb_rollout_gather_batch(h, field(host=1), 1, 1, None, 0, stream) == E_INVALID
    assert ops.ctx.launch_count == n0            # every refusal is decided before anything is launched
