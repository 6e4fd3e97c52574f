"""Restatement of the keyed sampling noise of Imagen.sample(seed=) (mi_randn_keyed), vectorised in numpy on uint64.

The generator, as the sampler specifies it:
  key      the image's 64-bit seed s as (lo32, hi32);
  counter  (q, label mod 2^32, kind, stage): element j of the image's flattened C*H*W data is lane j % 4 of quad q = j / 4;
           kind 0 'init', 1 'step', 2 'lowres', 3 'renoise', 4 'inpaint'; stage the U-Net number;
  bits     Philox4x32-10 (Salmon et al. 2011, Random123) with M = 0xD2511F53, 0xCD9E8D57 and W = 0x9E3779B9, 0xBB67AE85:
           ten rounds (hi0, lo0) = M0 * c0, (hi1, lo1) = M1 * c2, c <- (hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0), the key
           bumped by W between rounds;
  normals  Box-Muller on the pairs (x0, x1), (x2, x3): u = ((x_a >> 9) + 0.5) 2^-23, v = (x_b >> 8) 2^-24,
           z = sqrt(-2 ln u) (cos 2 pi v, sin 2 pi v).
`normals64` evaluates the last step in float64 from the same bits (with the quarter-turn reduction of cospi / sinpi, so
that their exact zeros stay exact); `normals32` is that rounded to fp32, the draw of the CPU emulation.
"""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
MASK32 = np.uint64(0xFFFFFFFF)
KINDS = {'init': 0, 'step': 1, 'lowres': 2, 'renoise': 3, 'inpaint': 4}


def philox4x32_10(ctr, key):
    """ctr: 4 uint64 arrays (32-bit words), key: 2 of them (broadcastable); returns the 4 output words as uint64."""
    c = [np.asarray(v, dtype=np.uint64) & MASK32 for v in ctr]
    k0, k1 = (np.asarray(v, dtype=np.uint64) & MASK32 for v in key)
    for rnd in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]                     # < 2^64: exact in uint64
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK32
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK32
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        if rnd < 9:
            k0, k1 = (k0 + W0) & MASK32, (k1 + W1) & MASK32
    return c


def bits(seed, n, kind, stage, label):
    """The 4 Philox words of each quad of one image's n elements: [ceil(n/4), 4] uint64."""
    nq = (n + 3) // 4
    s = int(seed)
    assert 0 <= s < 2 ** 64
    q = np.arange(nq, dtype=np.uint64)
    out = philox4x32_10((q, np.uint64(int(label) % 2 ** 32), np.uint64(kind), np.uint64(stage)),
                        (np.uint64(s & 0xFFFFFFFF), np.uint64(s >> 32)))
    return np.stack([np.broadcast_to(w, q.shape) for w in out], axis=1)


def _sincospi(a):
    """(sin(pi a), cos(pi a)) in float64 for a in [0, 2): reduce to r in [-1/4, 1/4] around the nearest quarter turn."""
    k = np.rint(2 * a)
    r = a - k / 2
    s, c = np.sin(np.pi * r), np.cos(np.pi * r)
    quad = k.astype(np.int64) % 4
    sin = np.choose(quad, [s, c, -s, -c])
    cos = np.choose(quad, [c, -s, -c, s])
    return sin, cos


def uv(x):
    """(u, v) of the pairs of the quads x [nq, 4]: [nq, 2] each, exact (float64 holds them as fp32 would)."""
    xa, xb = x[:, 0::2], x[:, 1::2]
    u = ((xa >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23
    v = (xb >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
    return u, v


def normals64(seed, n, kind, stage, label):
    """One image's n keyed normals in float64 from the generator's bits."""
    u, v = uv(bits(seed, n, kind, stage, label))
    rho = np.sqrt(-2.0 * np.log(u))
    sin, cos = _sincospi(2 * v)
    z = np.empty((u.shape[0], 4))
    z[:, 0::2] = rho * cos
    z[:, 1::2] = rho * sin
    return z.reshape(-1)[:n]


def normals32(seed, n, kind, stage, label):
    return normals64(seed, n, kind, stage, label).astype(np.float32)


def randn_keyed(seeds, n, kind, stage, labels, dtype=np.float64):
    """[B, n]: image b's draws for seeds[b] and labels[b] (an int for every image, or one per image)."""
    labels = np.broadcast_to(np.asarray(labels, dtype=object), (len(seeds),))
    f = normals64 if dtype == np.float64 else normals32
    return np.stack([f(s, n, kind, stage, lab) for s, lab in zip(seeds, labels)])


def ulp_bound():
    """The relative error bound of a kernel normal against the same formula in exact arithmetic, from the CUDA C
    Programming Guide's maximum ulp errors (no fast-math): logf 1 ulp, sqrtf 0 ulp (correctly rounded), sincospif 1 ulp
    for each of its two results (as cospif / sinpif), and 0.5 ulp for each rounded product.  With eps = 2^-24 (unit roundoff; 1 ulp <= 2 eps relative at normal
    results) and u, v, 2v and the factor -2 exact: logf gives ln u (1 + d1), |d1| <= 2 eps; the square root halves d1 and
    rounds once, so rho carries <= eps + eps; the trig value <= 2 eps; the product one more eps.  In total
    <= 5 eps (1 + O(eps)) < 6 eps = 2^-21.4, inside 2^-20 by a factor of 2.7."""
    eps = 2.0 ** -24
    rel = (2 * eps) / 2 + eps + 2 * eps + eps        # logf through the square root, sqrtf, cospif / sinpif, the product
    assert rel * (1 + 1e-6) < 6 * eps < 2.0 ** -20
    return 2.0 ** -20
