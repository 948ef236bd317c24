"""Float32 numpy model of one step of SAVi's belief update (BeliefPredictor.update,
ss_baselines/savi/models/belief_predictor.py:136-202), restated from its behaviour:

- env i is silent when its spectrogram is all zeros; ``dones[i]`` clears the env's state first;
- location: a sounding env takes ``base = (-p1, p0)`` from the prediction; without a state (or with
  ``current_pred_only``) the belief is ``base``, else ``(1-w) base + w to_base(state)``; the state becomes
  ``to_odom(belief)``.  A silent env reports ``to_base(state)``, or (10, 10) without a state;
- label: a sounding env's belief is the prediction's first 21 columns, or ``(1-w) label + w state``; the state becomes
  the belief.  A silent env reports the state, or 1/21 everywhere without one.

``to_base`` / ``to_odom`` are the planar frame changes between the episode's odometry frame and the agent's frame
(``pose`` = x, y, heading).  Every operation is one float32 numpy operation, so each product and sum is rounded on its
own; ``(1-w)`` and ``w`` enter as float32 scalars.  Also: the seeded sequences the golden recorder and the tests share.
"""
import numpy as np

F32 = np.float32
N_LABELS = 21


def _norm(x, y):
    return np.sqrt(x * x + y * y)


def odom_to_base(s, pose):
    dx, dy = s[0] - pose[0], s[1] - pose[1]
    theta = np.arctan2(dy, dx) - (-pose[2])
    d = _norm(dx, dy)
    return np.array([d * np.cos(theta), d * np.sin(theta)], dtype=F32)


def base_to_odom(a, pose):
    d = _norm(a[0], a[1])
    theta = np.arctan2(a[1], a[0]) + (-pose[2])
    return np.array([pose[0] + d * np.cos(theta), pose[1] + d * np.sin(theta)], dtype=F32)


def new_state(num_env):
    return dict(last_pg=np.zeros((num_env, 2), F32), loc_valid=np.zeros(num_env, bool),
                last_label=np.zeros((num_env, N_LABELS), F32), label_valid=np.zeros(num_env, bool))


def step(state, silent, pose, loc_pred, label_pred, dones, w, current_pred_only, loc_out=None, cat_out=None):
    """One ``update`` for B = len(silent) envs.  ``loc_pred`` / ``label_pred``: (B, >= 2) / (B, >= 21) float32 or None.
    Updates ``state`` in place; returns (loc_out (B, 2), cat_out (B, 21), decisions (B, 3) bool: silent, reset, first)
    where ``first`` = a sounding step with no state to average with.  Outputs not produced keep ``loc_out`` /
    ``cat_out`` (zeros when not given)."""
    B = len(silent)
    w1, w = F32(1.0 - w), F32(w)
    loc_out = np.zeros((B, 2), F32) if loc_out is None else loc_out.astype(F32).copy()
    cat_out = np.zeros((B, N_LABELS), F32) if cat_out is None else cat_out.astype(F32).copy()
    dec = np.zeros((B, 3), bool)
    for i in range(B):
        reset = dones is not None and bool(dones[i])
        dec[i, 0], dec[i, 1] = silent[i], reset
        for which in ("loc", "label"):
            pred = loc_pred if which == "loc" else label_pred
            if pred is None:
                continue
            vkey = "loc_valid" if which == "loc" else "label_valid"
            if reset:
                state[vkey][i] = False
            has = bool(state[vkey][i])
            if not silent[i]:
                dec[i, 2] = not has
                use_pred = not has or current_pred_only
                if which == "loc":
                    p = pose[i].astype(F32)
                    base = np.array([-F32(pred[i, 1]), F32(pred[i, 0])], dtype=F32)
                    avg = base if use_pred else w1 * base + w * odom_to_base(state["last_pg"][i], p)
                    state["last_pg"][i] = base_to_odom(avg, p)
                    loc_out[i] = avg
                else:
                    lab = pred[i, :N_LABELS].astype(F32)
                    avg = lab if use_pred else w1 * lab + w * state["last_label"][i]
                    state["last_label"][i] = avg
                    cat_out[i] = avg
                state[vkey][i] = True
            elif which == "loc":
                loc_out[i] = odom_to_base(state["last_pg"][i], pose[i].astype(F32)) if has else (10.0, 10.0)
            else:
                cat_out[i] = state["last_label"][i] if has else F32(1.0 / 21.0)
    return loc_out, cat_out, dec


def location_bound(scale):
    """Largest |difference| allowed between two float32 evaluations of the location belief that differ only in their
    sin / cos / atan2 (numpy's vs CUDA's full-precision sinf / cosf / atan2f), for poses, beliefs and states of size
    at most ``scale`` (>= 1) and headings in [-pi, pi).

    One frame change: atan2 is within 3 ulp on the device and 1 on the host, and its sum with the heading (|.| < 2 pi,
    ulp 2^-21) can round the other way once more: 5 ulp of 2 pi = 20 * 2^-23 rad.  Over a distance d <= 2 scale that
    moves the point by 40 * 2^-23 scale; sin / cos (2 ulp on the device, 1 on the host) add 3 * 2^-24 * d, and the
    product and the sum with the pose can each round the other way (ulp <= 2^-23 * 2 scale): about 50 * 2^-23 scale.
    A step changes frames twice (odom_to_base, base_to_odom), and the state carries a share w <= 1/2 of the previous
    error on (both changes are isometries), so the error stays below 2 * 2 * 50 * 2^-23 * scale.  Rounded up:
    256 * 2^-23 * scale, about 3.1e-5 * scale."""
    return 256.0 * 2.0 ** -23 * max(1.0, float(scale))


def make_sequence(seed, T, B, loc_cols=2, p_silent=0.2, p_done=0.06):
    """Seeded rollout inputs: ``silent`` (T, B) bool, with every env silent on its first step and after some dones,
    ``dones`` (T, B), a random-walk ``pose`` (T, B, 4) float32 (x, y, heading in [-pi, pi), time), location
    predictions (T, B, loc_cols) and label scores (T, B, 21), float32."""
    rng = np.random.default_rng(seed)
    silent = rng.random((T, B)) < p_silent
    dones = rng.random((T, B)) < p_done
    silent[0] = True
    silent[1:][dones[:-1]] |= rng.random(int(dones[:-1].sum())) < 0.5
    pose = np.zeros((T, B, 4), F32)
    xy = rng.normal(0, 2, (B, 2))
    head = rng.uniform(-np.pi, np.pi, B)
    for t in range(T):
        if t:
            head = (head + rng.choice([-np.pi / 18, 0.0, np.pi / 18], B) + np.pi) % (2 * np.pi) - np.pi
            xy = xy + 0.25 * np.stack([np.cos(head), np.sin(head)], 1) * (rng.random(B) < 0.7)[:, None]
            xy[dones[t - 1]] = rng.normal(0, 2, (int(dones[t - 1].sum()), 2))
        pose[t, :, :2], pose[t, :, 2], pose[t, :, 3] = xy, head, t
    loc_pred = rng.normal(0, 4, (T, B, loc_cols)).astype(F32)
    label_pred = rng.normal(0, 1, (T, B, N_LABELS)).astype(F32)
    return dict(silent=silent, dones=dones, pose=pose, loc_pred=loc_pred, label_pred=label_pred)


def make_spectrograms(silent, shape, seed):
    """(len(silent),) + shape float32: zeros for silent envs, log1p-like non-negative values (with some exact zeros)
    otherwise."""
    rng = np.random.default_rng(seed)
    x = rng.random((len(silent),) + tuple(shape), dtype=F32)
    x[x < 0.3] = 0
    x[np.asarray(silent)] = 0
    return x
