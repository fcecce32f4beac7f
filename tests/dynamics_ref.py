"""An independent float64 restatement of the step's wheel path (DESIGN.md §4): the action map, the clip, the command
delay line and one step of the DB18 model.  Test infrastructure, numpy + scipy only.

It is written differently from the kernel and the C oracle on purpose.  The pose update is the matrix exponential of
the twist, `q' = q · expm(dt · [[0, -w', u'], [w', 0, 0], [0, 0, 0]])`, evaluated by scipy, not the closed form
(sin a / a, (1 - cos a) / a, with a Taylor branch below |a| = 1e-9) that both of them use.  So the closed form and its
branch are checked against something that shares neither.
"""
import numpy as np
from scipy.linalg import expm

MODEL_KEYS = ("u1", "u2", "u3", "w1", "w2", "w3", "uar", "ual", "war", "wal")


def action_map(vel, steer, wheel_dist, gain=1.0, trim=0.0, radius=0.0318, k=27.0, limit=1.0):
    """DuckietownEnv.step's [vel, steering] -> (left, right) wheel duty, clamped to +-limit."""
    omega_r = (vel + 0.5 * steer * wheel_dist) / radius
    omega_l = (vel - 0.5 * steer * wheel_dist) / radius
    u_r = omega_r * ((gain + trim) / k)
    u_l = omega_l * ((gain - trim) / k)
    return float(np.clip(u_l, -limit, limit)), float(np.clip(u_r, -limit, limit))


def clip_duty(lr):
    """Simulator.step's np.clip(action, -1, 1), which the model applies once more to the duty it is handed."""
    return np.clip(np.asarray(lr, np.float64), -1.0, 1.0)


def delay_push(line, cmd, d):
    """The command delay line of depth d (oldest first): returns (the duty that acts now, the line after the push)."""
    if d == 0:
        return np.asarray(cmd, np.float64), np.asarray(line, np.float64).copy()
    line = np.asarray(line, np.float64)
    out = line.copy()
    out[:d - 1] = line[1:d]
    out[d - 1] = cmd
    return line[0].copy(), out


def db18_step(x, y, theta, u, w, duty_lr, model, trim, dt):
    """One step of the DB18 model from cartesian pose (x, y, theta) and velocities (u, w) under wheel duty
    (left, right): returns (x, y, theta, u, w).  theta is returned unwrapped, theta + dt·w', as the state keeps it."""
    p = model
    l, r = clip_duty(duty_lr)
    uar, ual = p["uar"] * (1 + trim), p["ual"] * (1 - trim)
    war, wal = p["war"] * (1 + trim), p["wal"] * (1 - trim)
    u1 = u + dt * (-p["u1"] * u - p["u2"] * w + p["u3"] * w * w + uar * r + ual * l)
    w1 = w + dt * (-p["w1"] * w - p["w2"] * u - p["w3"] * u * w + war * r - wal * l)
    c, s = np.cos(theta), np.sin(theta)
    q = np.array([[c, -s, x], [s, c, y], [0.0, 0.0, 1.0]])
    twist = np.array([[0.0, -w1, u1], [w1, 0.0, 0.0], [0.0, 0.0, 0.0]])
    q1 = q @ expm(dt * twist)
    return q1[0, 2], q1[1, 2], theta + dt * w1, u1, w1


# Test configurations of the model.  ALL sets every constant non-zero and distinct, with left and right gains that
# differ.  TURN has w2 = 0: the turn a = dt·w' of the step then follows w with no large constant term beside it, so a
# state can be chosen whose a lands on a given double exactly (`w_for_turn`).
MODEL_ALL = dict(u1=4.3, u2=0.37, u3=0.061, w1=3.7, w2=0.53, w3=0.29, uar=1.62, ual=1.41, war=16.3, wal=13.9)
MODEL_TURN = dict(MODEL_ALL, w2=0.0)


def turn_values():
    """The turns a = dt·w' where the closed form's branches meet or its terms lose precision: 0, +-1e-12, the 1e-9
    Taylor threshold and three ulps either side of it (both signs), 1e-6, 1 and +-pi."""
    out = [0.0, 1e-12, -1e-12, 1e-6, 1.0, np.pi, -np.pi]
    for sign in (1.0, -1.0):
        v = sign * 1e-9
        out.append(v)
        lo = hi = v
        for _ in range(3):
            lo, hi = np.nextafter(lo, 0.0), np.nextafter(hi, sign * np.inf)
            out += [float(lo), float(hi)]
    return out


def w_for_turn(a, u, model, trim, dt):
    """A starting w whose step turns by exactly `a` (or as near as a double allows) when the duty acting is (0, 0) and
    the speed is u, in the float64 arithmetic of the kernel and the oracle (same operations, same order):
    dw = -w1·w - w2·u - w3·u·w + (war·r - wal·l); a = dt·(w + dt·dw).  Returns (w, the a it gives)."""
    p = model
    war, wal = p["war"] * (1.0 + trim), p["wal"] * (1.0 - trim)

    def turn(w):
        dw = -p["w1"] * w - p["w2"] * u - p["w3"] * u * w + (war * 0.0 - wal * 0.0)
        return dt * (w + dt * dw)

    w = a / (dt * (1.0 - dt * (p["w1"] + p["w3"] * u))) if a else 0.0
    best = w
    for direction in (np.inf, -np.inf):
        c = w
        for _ in range(256):
            if abs(turn(c) - a) < abs(turn(best) - a):
                best = c
            if turn(c) == a:
                return float(c), a
            c = np.nextafter(c, direction)
    return float(best), turn(best)
