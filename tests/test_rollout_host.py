"""CPU tests of the device rollout storage (soundspaces_b200/rollout.py): the stand-ins against the reference golden,
layout recognition and every reason a storage does not qualify, the originals running for CPU storage, patch
idempotence, the generator's RNG use and assertion, ``patch_ppo`` and DD-PPO's instance override, and the ABI."""
import os
import re
import types

import numpy as np
import pytest
import torch

import rollout_models as rm
from soundspaces_b200 import _lib
from soundspaces_b200 import rollout as ro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "rollout_golden.npz")
STAND_INS = dict(common=rm.CommonRolloutStorage, savi=rm.SaviRolloutStorage)


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _patched_classes():
    """Patched subclasses of the stand-ins (the stand-ins themselves stay eager)."""
    classes = {k: type("Patched" + v.__name__, (v,), {}) for k, v in STAND_INS.items()}
    for cls in classes.values():
        ro.patch_rollout_storage(cls)
    ppo = ro.patch_ppo(type("PatchedPPO", (rm.PPO,), {}))
    return classes, ppo


def _check(res, golden, prefix):
    keys = [k for k in golden if k.startswith(prefix + "/")]
    assert keys and len(keys) == len(res)
    for k in keys:
        got = res[k[len(prefix) + 1:]]
        assert got.dtype == golden[k].dtype and got.shape == golden[k].shape, k
        assert np.array_equal(got.view(np.uint8), golden[k].view(np.uint8)), k


@pytest.mark.parametrize("use_gae", [True, False])
@pytest.mark.parametrize("name", sorted(rm.SCRIPTS))
def test_stand_ins_match_reference_golden(golden, name, use_gae):
    res = rm.run_script(rm.SCRIPTS[name], STAND_INS, rm.PPO, use_gae)
    _check(res, golden, rm.golden_key(name, use_gae))


def test_golden_covers_what_the_kernels_must_reproduce(golden):
    savi = rm.golden_key("savi", True)
    held = golden[f"{savi}/0/state/em_masks_mem"].sum(1)
    assert held.max() == rm.SCRIPTS["savi"]["em"][1]              # the memory reaches capacity
    masks = golden[f"{rm.golden_key('common', True)}/0/state/masks"][1:, :, 0]
    assert (masks == 0).any() and len({tuple(np.nonzero(masks[:, e] == 0)[0]) for e in range(4)}) > 1
    assert golden[f"{rm.golden_key('common', True)}/0/mb2/actions"].dtype == np.int64
    for m in rm.MINI_BATCHES:
        assert golden[f"{savi}/0/mb{m}/em_store"].shape[0] == m


@pytest.mark.parametrize("use_gae", [True, False])
@pytest.mark.parametrize("name", sorted(rm.SCRIPTS))
def test_patched_cpu_storage_runs_the_originals(golden, name, use_gae):
    classes, ppo = _patched_classes()
    res = rm.run_script(rm.SCRIPTS[name], classes, ppo, use_gae)
    _check(res, golden, rm.golden_key(name, use_gae))


def _storage(name="savi", **kw):
    script = dict(rm.SCRIPTS[name], **kw)
    return rm.make_storage(script, STAND_INS)


def test_layout_recognition_and_every_reason():
    cpu = torch.device("cpu")
    assert ro.rollout_layout_error(_storage()) == "the storage is on the CPU"
    for name in rm.SCRIPTS:
        assert ro._layout_error(_storage(name), cpu) == ""
    st = _storage()
    st.rewards = st.rewards.transpose(0, 1).contiguous().transpose(0, 1)
    assert ro._layout_error(st, cpu) == "rewards is not contiguous"
    st = _storage()
    st.em.__class__ = rm.ExternalMemoryVaried
    assert "ExternalMemoryVaried" in ro._layout_error(st, cpu)
    st = _storage()
    st.em.idx = torch.zeros(4, dtype=torch.long)
    assert "idx" in ro._layout_error(st, cpu)
    st = _storage()
    st.value_preds = st.value_preds.double()
    assert "value_preds is not float32" in ro._layout_error(st, cpu)
    st = _storage()
    st.masks = st.masks[:, :3].contiguous()
    assert "masks has shape" in ro._layout_error(st, cpu)
    st = _storage("common")
    st.prev_actions = st.prev_actions.float()
    assert "prev_actions" in ro._layout_error(st, cpu)
    assert "on cpu" not in ro._layout_error(_storage(), torch.device("meta"))   # every tensor must be on the device
    assert "is not a tensor on meta" in ro._layout_error(_storage(), torch.device("meta"))
    for kw, what in ((dict(S=ro.MAX_STEPS + 1), "steps"),
                     (dict(sensors={f"s{i}": (1,) for i in range(ro.MAX_SENSORS + 1)}), "sensors"),
                     (dict(em=(ro.MAX_MEMORY + 1, 5, 1)), "slots"),
                     (dict(em=(11, 12, 3)), "capacity")):
        assert what in ro._layout_error(_storage(**kw), cpu), kw
    st = _storage()
    st.em_masks = st.em_masks[:, :, :5].contiguous()
    assert "em_masks" in ro._layout_error(st, cpu)
    # a subclass whose memory keeps ExternalMemory's insert still qualifies
    st = _storage()
    st.em.__class__ = type("Sub", (rm.ExternalMemory,), {})
    assert ro._layout_error(st, cpu) == ""


def test_patch_is_idempotent_and_keeps_the_originals():
    cls = type("P", (rm.SaviRolloutStorage,), {})
    ro.patch_rollout_storage(cls)
    first = {n: getattr(cls, n) for n in ("insert", "compute_returns", "recurrent_generator", "after_update")}
    ro.patch_rollout_storage(cls)
    for n, fn in first.items():
        assert getattr(cls, n)._ssb_original is getattr(rm.SaviRolloutStorage, n)
        assert fn._ssb_original is getattr(cls, n)._ssb_original
    em = type("E", (rm.ExternalMemory,), {})
    ro.patch_external_memory(em)
    ro.patch_external_memory(em)
    assert em.insert._ssb_original is rm.ExternalMemory.insert
    ppo = type("Q", (rm.PPO,), {})
    ro.patch_ppo(ppo)
    ro.patch_ppo(ppo)
    assert ppo.get_advantages._ssb_original is rm.PPO.get_advantages


def test_patched_memory_keeps_its_insert_recognised():
    cls = type("E2", (rm.ExternalMemory,), {})
    ro.patch_external_memory(cls)
    st = _storage()
    st.em.__class__ = cls
    assert ro._layout_error(st, torch.device("cpu")) == ""


def test_generator_rng_use_and_assertion():
    classes, _ = _patched_classes()
    for kind in ("common", "savi"):
        script = rm.SCRIPTS["common" if kind == "common" else "savi"]
        st = rm.make_storage(script, classes)
        if kind == "savi":
            st.step = script["S"]
        adv = torch.zeros(script["S"], script["N"], 1)
        torch.manual_seed(5)
        list(st.recurrent_generator(adv, 2))
        after = torch.get_rng_state()
        torch.manual_seed(5)
        torch.randperm(script["N"])
        assert torch.equal(after, torch.get_rng_state())
        with pytest.raises(AssertionError, match=r"Trainer requires the number of processes \(4\) to be greater than "
                                                  r"or equal to the number of trainer mini batches \(5\)\."):
            next(st.recurrent_generator(adv, 5))


def test_ppo_patch_leaves_the_distributed_override_alone():
    ppo_cls = ro.patch_ppo(type("PPOD", (rm.PPO,), {}))
    agent = ppo_cls()
    called = []

    def distributed(rollouts):
        called.append(rollouts)
        return "distributed"

    agent.get_advantages = distributed          # what DD-PPO's init_distributed does
    st = _storage("common")
    assert agent.get_advantages(st) == "distributed" and called == [st]
    plain = ppo_cls(use_normalized_advantage=False)
    st.returns.normal_()
    assert torch.equal(plain.get_advantages(st), st.returns[:-1] - st.value_preds[:-1])
    assert torch.equal(ppo_cls().get_advantages(st), rm.PPO().get_advantages(st))    # CPU: the original


def _header_params(name):
    with open(os.path.join(ROOT, "include", "ssb200.h")) as f:
        text = f.read()
    m = re.search(r"\bint " + name + r"\(([^;]*)\);", text)
    assert m, name
    return [p.strip() for p in m.group(1).split(",")]


@pytest.mark.parametrize("name", ["ssb_rollout_insert_batch", "ssb_rollout_returns_batch", "ssb_rollout_gather_batch"])
def test_abi_prototypes_match_the_header(name):
    assert len(_lib.EXPORTS[name][1]) == len(_header_params(name))


def test_abi_structs_match_the_header():
    import ctypes
    assert ctypes.sizeof(_lib.RolloutField) == 56
    assert ctypes.sizeof(_lib.RolloutMemory) == 56
    assert ro.MAX_FIELDS == 32 and ro.MAX_COLS == 256
    with open(os.path.join(ROOT, "include", "ssb200.h")) as f:
        text = f.read()
    for macro, value in (("SSB_ROLLOUT_MAX_FIELDS", ro.MAX_FIELDS), ("SSB_ROLLOUT_MAX_COLS", ro.MAX_COLS),
                         ("SSB_ROLLOUT_MAX_ENVS", ro.MAX_ENVS), ("SSB_ROLLOUT_MAX_STEPS", ro.MAX_STEPS),
                         ("SSB_ROLLOUT_MAX_MEMORY", ro.MAX_MEMORY)):
        assert re.search(rf"#define {macro} {value}\b", text), macro


def test_advantages64_is_the_reference_formula():
    r = np.random.default_rng(0)
    ret, vp = r.standard_normal((5, 3, 1)).astype(np.float32), r.standard_normal((5, 3, 1)).astype(np.float32)
    st = types.SimpleNamespace(returns=torch.from_numpy(ret), value_preds=torch.from_numpy(vp))
    got = rm.PPO().get_advantages(st).numpy()
    assert np.abs(got - rm.advantages64(ret, vp)).max() < 1e-5
