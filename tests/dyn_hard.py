"""TEST INFRASTRUCTURE — hard model and state families for the rigid-body kernels (libtoppra_b200_dyn.so).

`rnea_ref.random_tree` draws bushy trees of well-behaved bodies.  The families here go to the other ends, within the
kernels' limits (nv <= 16 bodies, P <= 16 points, H <= 16 humans):

* `serial_chain(rng, nv)`: body k on body k - 1, so a frame on the last body walks all nv bodies from the root; every
  fourth joint is prismatic on a random axis.
* `star(rng, nv)`: every body on the base, bodies 0 and 1 sliders along the base's x and z axes.  `broom(rng)`: an 8-deep chain
  that ends in 8 leaves on its last body.
* `badly_scaled(rng, nv)`: a serial chain whose masses fall from 1e3 to 1e-3 kg down the chain, whose link offsets are
  log-uniform in 1e-3..2 m and whose inertias are rods (one principal moment 1e-6 of the other two).
* `planar(rng, nv, kind)`: every joint axis along z.  kind "revolute": a planar arm whose links all lie along x at
  q = 0 (a stretched, singular pose); "prismatic": an all-prismatic chain on random axes (no rotation at all);
  "rp": revolute about z alternating with prismatic along x, in the plane.
* `states(rng, nv)`: the points (q, qd, qdd) every case is evaluated at: fast motion (qd up to 50 rad/s, where the
  velocity-product terms are about 1e3 times gravity), wound-up joints (|q| up to 1e3 rad, the sin/cos argument
  reduction) and the stretched pose q = 0.

Each family returns a packed model (include/toppra_b200_dyn.h).  `CASES` is the list the fixture
tests/golden/dyn_hard_trees.npz is made of; `case_model(name)` rebuilds a case's model from its seed."""
import numpy as np

BODY = 27
MAX_BODIES = 16


def _rotation(rng):
    Q, _ = np.linalg.qr(rng.randn(3, 3))
    return Q * np.sign(np.linalg.det(Q))


def _unit(rng):
    a = rng.randn(3)
    return a / np.linalg.norm(a)


def _rz(t):
    c, s = np.cos(t), np.sin(t)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def _inertia6(I):
    return [I[0, 0], I[0, 1], I[0, 2], I[1, 1], I[1, 2], I[2, 2]]


def _physical_inertia(rng, scale):
    """A random rotational inertia with principal moments in scale * [0.1, 1] that meet the triangle inequalities."""
    mom = rng.uniform(0.1, 1.0, 3) * scale
    mom[2] = rng.uniform(abs(mom[0] - mom[1]) + 0.01 * scale, mom[0] + mom[1] - 0.01 * scale)
    P = _rotation(rng)
    return P @ np.diag(mom) @ P.T


def _empty(nv, gravity):
    if not 1 <= nv <= MAX_BODIES:
        raise ValueError("nv = %d outside 1..%d" % (nv, MAX_BODIES))
    packed = np.zeros(3 + BODY * nv)
    packed[:3] = gravity
    return packed, packed[3:].reshape(nv, BODY)


def _generic_body(rng, bd, parent, prismatic):
    bd[0] = parent
    bd[1] = 1.0 if prismatic else 0.0
    bd[2:5] = _unit(rng)
    bd[5:14] = _rotation(rng).reshape(9)
    bd[14:17] = rng.randn(3) * 0.3
    bd[17] = rng.uniform(0.1, 5.0)
    bd[18:21] = rng.randn(3) * 0.1
    bd[21:27] = _inertia6(_physical_inertia(rng, 0.1))


def _tree(rng, parents, gravity):
    packed, b = _empty(len(parents), gravity)
    for k, par in enumerate(parents):
        _generic_body(rng, b[k], par, k % 4 == 2)
    return packed


def serial_chain(rng, nv, gravity=(0.0, 0.0, -9.81)):
    return _tree(rng, [k - 1 for k in range(nv)], gravity)


def star(rng, nv=16, gravity=(0.0, 0.0, -9.81)):
    """Every body on the base.  Bodies 0 and 1 are sliders along the base's x and z axes from its origin (E = I, r = 0),
    so that their origins are (q0, 0, 0) and (0, 0, q1), exactly, at every q."""
    packed = _tree(rng, [-1] * nv, gravity)
    b = packed[3:].reshape(nv, BODY)
    for k, axis in ((0, (1.0, 0.0, 0.0)), (1, (0.0, 0.0, 1.0)))[:nv]:
        b[k, 1], b[k, 2:5], b[k, 5:14], b[k, 14:17] = 1.0, axis, np.eye(3).reshape(9), 0.0
    return packed


def broom(rng, depth=8, leaves=8, gravity=(0.0, 0.0, -9.81)):
    return _tree(rng, [k - 1 for k in range(depth)] + [depth - 1] * leaves, gravity)


def badly_scaled(rng, nv=16, gravity=(0.0, 0.0, -9.81)):
    """Masses 1e3 .. 1e-3 kg decreasing down a serial chain, offsets log-uniform in 1e-3 .. 2 m (the first and last
    links at the two ends), rod-like inertias m L^2 / 12 with the rod's own moment 1e-6 of that."""
    packed, b = _empty(nv, gravity)
    mass = np.logspace(3, -3, nv) if nv > 1 else np.array([1e3])
    length = 10.0 ** rng.uniform(-3, np.log10(2.0), nv)
    length[0], length[-1] = 2.0, 1e-3
    for k in range(nv):
        bd = b[k]
        _generic_body(rng, bd, k - 1, k % 5 == 3)
        bd[14:17] = _unit(rng) * length[k]
        bd[17] = mass[k]
        bd[18:21] = rng.randn(3) * 0.3 * length[k]
        I = mass[k] * length[k] ** 2 / 12.0
        P = _rotation(rng)
        bd[21:27] = _inertia6(P @ np.diag([I, I, I * 1e-6]) @ P.T)       # a rod: I <= I + 1e-6 I, the triangle kept
    return packed


def planar(rng, nv=16, kind="revolute", gravity=(0.0, -9.81, 0.0)):
    """Every joint axis along z (see the module docstring for the three kinds)."""
    packed, b = _empty(nv, gravity)
    for k in range(nv):
        bd = b[k]
        bd[0] = k - 1
        L = rng.uniform(0.05, 0.4)
        if kind == "revolute":
            bd[1], bd[2:5], E = 0.0, (0.0, 0.0, 1.0), np.eye(3)
            bd[14:17] = (L, 0.0, 0.0) if k else (0.0, 0.0, 0.0)
        elif kind == "prismatic":
            bd[1], bd[2:5], E = 1.0, _unit(rng), _rotation(rng)
            bd[14:17] = rng.randn(3) * 0.2
        elif kind == "rp":
            bd[1], bd[2:5] = (0.0, (0.0, 0.0, 1.0)) if k % 2 == 0 else (1.0, (1.0, 0.0, 0.0))
            E = _rz(rng.uniform(-np.pi, np.pi))
            bd[14:17] = (L, rng.uniform(-0.1, 0.1), 0.0)
        else:
            raise ValueError(kind)
        bd[5:14] = E.reshape(9)
        bd[17] = rng.uniform(0.1, 5.0)
        bd[18:21] = (0.5 * L, rng.uniform(-0.02, 0.02), rng.uniform(-0.02, 0.02))
        bd[21:27] = _inertia6(_physical_inertia(rng, 0.05))
    return packed


STATE_KINDS = ("fast", "wound", "stretched")


def states(rng, nv):
    """(q, qd, qdd), each (3, nv): one point per kind of STATE_KINDS."""
    q = np.stack([rng.uniform(-np.pi, np.pi, nv), rng.uniform(-1e3, 1e3, nv), np.zeros(nv)])
    qd = np.stack([rng.uniform(-50, 50, nv), rng.uniform(-2, 2, nv), rng.uniform(-1, 1, nv)])
    qdd = np.stack([rng.uniform(-200, 200, nv), rng.uniform(-5, 5, nv), rng.uniform(-3, 3, nv)])
    return q, qd, qdd


# name -> (family, seed, builder(rng)).  Families with 16 bodies also have a small member, so that one case per family
# can be recomputed at 50 digits in a test.
CASES = {
    "chain1": ("serial_chain", 101, lambda rng: serial_chain(rng, 1)),
    "chain8": ("serial_chain", 108, lambda rng: serial_chain(rng, 8)),
    "chain15_zero_g": ("serial_chain", 115, lambda rng: serial_chain(rng, 15, gravity=(0.0, 0.0, 0.0))),
    "chain16": ("serial_chain", 116, lambda rng: serial_chain(rng, 16)),
    "star4": ("star", 204, lambda rng: star(rng, 4)),
    "star16": ("star", 216, lambda rng: star(rng, 16)),
    "broom": ("broom", 316, lambda rng: broom(rng)),
    "broom_small": ("broom", 305, lambda rng: broom(rng, 3, 2)),
    "scaled5": ("badly_scaled", 405, lambda rng: badly_scaled(rng, 5)),
    "scaled16": ("badly_scaled", 416, lambda rng: badly_scaled(rng, 16)),
    "planar_r4": ("planar", 504, lambda rng: planar(rng, 4, "revolute")),
    "planar_r16": ("planar", 516, lambda rng: planar(rng, 16, "revolute")),
    "planar_p16": ("planar", 526, lambda rng: planar(rng, 16, "prismatic")),
    "planar_rp16": ("planar", 536, lambda rng: planar(rng, 16, "rp")),
}
PIN_CASES = ("chain8", "star4", "broom_small", "scaled5", "planar_r4")   # the small member of each family


def case_model(name):
    """(packed model, q, qd, qdd) of a case, from its seed."""
    _, seed, build = CASES[name]
    rng = np.random.RandomState(seed)
    packed = build(rng)
    return (packed,) + states(rng, (len(packed) - 3) // BODY)


def depth(packed, body):
    """The number of bodies on the root chain of `body` (itself included)."""
    n = 0
    while body >= 0:
        n += 1
        body = int(packed[3 + BODY * body])
    return n


def deepest(packed):
    """The highest-numbered body of greatest depth: where a frame walks the longest chain."""
    nv = (len(packed) - 3) // BODY
    d = [depth(packed, k) for k in range(nv)]
    return max(range(nv), key=lambda k: (d[k], k))
