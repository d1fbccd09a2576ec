"""Reference of the open boundaries (DESIGN.md section 2.6): the emitter's axes and schedule in float64, the emitted layers and the
sink test in float32, each evaluated in the order include/sphk.h states, so that the library's results can be compared bit for
bit."""
import numpy as np

F = np.float32


def axes(origin, direction, speed, spacing, width, height):
    """(d, e1, e2) as float32[3] each: d normalised in double; e1 = normalize(d x y^), or normalize(d x x^) when |d . y^| > 0.9;
    e2 = e1 x d; all in double, rounded once"""
    d = np.asarray(direction, np.float32).astype(np.float64)
    d = d / np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
    c = np.array([0.0, d[2], -d[1]]) if abs(d[1]) > 0.9 else np.array([-d[2], 0.0, d[0]])
    e1 = c / np.sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2])
    e2 = np.array([e1[1] * d[2] - e1[2] * d[1], e1[2] * d[0] - e1[0] * d[2], e1[0] * d[1] - e1[1] * d[0]])
    return d.astype(F), e1.astype(F), e2.astype(F)


def advance(carry: float, speed, spacing, dt, max_layers: int):
    """one step of the schedule: (new carry, scheduled layers, offsets of the first min(scheduled, max_layers) as float32)"""
    s = float(F(spacing))
    c = carry + float(F(speed)) * float(F(dt))
    offsets, k = [], 0
    while c >= s:
        if k < max_layers:
            offsets.append(F(c - s))
        c -= s
        k += 1
    return c, k, np.array(offsets, F)


def layers(e: dict, offsets) -> tuple:
    """positions (k W H, 3) and velocity (3,) of the layers at `offsets`, slot k W H + b W + a, float32 without contraction"""
    d, e1, e2 = axes(**e)
    W, H = int(e["width"]), int(e["height"])
    o, s, u = np.asarray(e["origin"], F), F(e["spacing"]), F(e["speed"])
    a = np.tile(np.arange(W, dtype=F), H)
    b = np.repeat(np.arange(H, dtype=F), W)
    ta = (a - F(0.5) * F(W - 1)) * s
    tb = (b - F(0.5) * F(H - 1)) * s
    out = []
    for delta in np.asarray(offsets, F):
        x = o[None, :] + ta[:, None] * e1[None, :]
        x = x + tb[:, None] * e2[None, :]
        x = x + F(delta) * d[None, :]
        out.append(x.astype(F))
    pos = np.concatenate(out, 0) if out else np.zeros((0, 3), F)
    return pos, (u * d).astype(F)


def sink_mask(pos, boxes) -> np.ndarray:
    """particles with lo <= x < hi on all three axes of some box {lo.xyz, hi.xyz} (float32 compares)"""
    pos = np.asarray(pos, F)
    m = np.zeros(pos.shape[0], bool)
    for b in np.asarray(boxes, F).reshape(-1, 6):
        m |= ((pos >= b[:3]) & (pos < b[3:])).all(1)
    return m


def tap_and_drain(box, block, origin, tap, drain, spacing=F(0.02)):
    """sph_headless --tap SPEED / --drain SIDE: the emitter dict and the sink box, float32 as the app computes them"""
    box, origin = [F(x) for x in box], [F(x) for x in origin]
    half = F(0.5) * F(spacing)
    e = {"origin": [origin[0] + half * F(block[0] - 1), F(0.85) * box[1], origin[2] + half * F(block[2] - 1)],
         "direction": [0.0, -1.0, 0.0], "speed": F(tap), "spacing": F(spacing), "width": 8, "height": 8}
    sink = np.array([0.0, 0.0, 0.0, F(drain), F(0.05) * box[1], F(drain)], F)
    return e, sink
