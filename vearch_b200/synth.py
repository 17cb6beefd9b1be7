"""Seeded synthetic inputs for tests and bench (SURVEY.md 8d).

SIFT-shaped: d-dim mixture of Gaussian clusters with ANISOTROPIC per-cluster noise (a quarter
of the dimensions carry most of the variance, like SIFT's gradient-histogram bins), clipped to
[0, 218] and rounded to integers stored as fp32 -- every partial sum of squared differences is
then exactly representable in fp32 (d * 218^2 < 2^24 for d <= 353), so distances are independent
of summation order and GPU-vs-oracle parity on this data is bit-exact.
Embedding-shaped: same mixture, unrounded, L2-normalised (cosine == inner product).
"""
import numpy as np

HI_SIGMA, LO_SIGMA, HI_FRAC = 24.0, 3.0, 0.25


def _centers_np(n_clusters, d, centers_seed):
    rng_c = np.random.default_rng(centers_seed)
    centers = rng_c.uniform(0, 128, size=(n_clusters, d)).astype(np.float32)
    centers *= (rng_c.random((n_clusters, d)) < 0.5)
    scale = np.where(rng_c.random((n_clusters, d)) < HI_FRAC, HI_SIGMA, LO_SIGMA).astype(np.float32)
    return centers, scale


def sift_like(n, d=128, seed=1234, n_clusters=256, centers_seed=99, rounded=True):
    """rounded=False: the same mixture left un-rounded (every mantissa bit in use) -- the float-valued parity set"""
    centers, scale = _centers_np(n_clusters, d, centers_seed)
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, n_clusters, size=n)
    x = centers[lab] + rng.normal(0, 1, size=(n, d)).astype(np.float32) * scale[lab]
    if not rounded:
        return (np.clip(x, 0, 218) * np.float32(1.0 / 3.0)).astype(np.float32)
    return np.clip(np.rint(x), 0, 218).astype(np.float32)


def embed_like(n, d=768, seed=1234, n_clusters=256, centers_seed=99, sigma=0.6):
    rng_c = np.random.default_rng(centers_seed)
    centers = rng_c.normal(0, 1, size=(n_clusters, d)).astype(np.float32)
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, n_clusters, size=n)
    x = centers[lab] + rng.normal(0, sigma, size=(n, d)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return x.astype(np.float32)


def sift_like_torch(n, d, seed, device, n_clusters=4096, centers_seed=99, chunk=1 << 20):
    """Same family as sift_like, generated on `device` with torch (bench sizes)."""
    import torch
    gc = torch.Generator(device=device)
    gc.manual_seed(centers_seed)
    centers = torch.rand((n_clusters, d), generator=gc, device=device) * 128.0
    centers = centers * (torch.rand((n_clusters, d), generator=gc, device=device) < 0.5)
    hi = torch.rand((n_clusters, d), generator=gc, device=device) < HI_FRAC
    scale = torch.where(hi, torch.tensor(HI_SIGMA, device=device), torch.tensor(LO_SIGMA, device=device))
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    out = torch.empty((n, d), dtype=torch.float32, device=device)
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        lab = torch.randint(0, n_clusters, (e - s,), generator=g, device=device)
        x = centers[lab] + torch.randn((e - s, d), generator=g, device=device) * scale[lab]
        out[s:e] = torch.clamp(torch.round(x), 0, 218)
    return out


def embed_like_torch(n, d, seed, device, n_clusters=4096, centers_seed=99, sigma=0.6, chunk=1 << 18):
    import torch
    gc = torch.Generator(device=device)
    gc.manual_seed(centers_seed)
    centers = torch.randn((n_clusters, d), generator=gc, device=device)
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    out = torch.empty((n, d), dtype=torch.float32, device=device)
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        lab = torch.randint(0, n_clusters, (e - s,), generator=g, device=device)
        x = centers[lab] + torch.randn((e - s, d), generator=g, device=device) * sigma
        out[s:e] = x / x.norm(dim=1, keepdim=True)
    return out


# ---- a harder SIFT-shaped family (VERDICT r1 item 8) ------------------------------------------------------
# Points near a `latent`-dimensional linear manifold (x = 100 + 3 W z + noise, integer-rounded like sift_like), z from
# `n_comp` OVERLAPPING Gaussians with Zipf weights: k-means cells cut through dense regions, true neighbours straddle
# lists (recall rises with nprobe instead of saturating at the first probes) and list lengths are heavy-tailed.
def _hard_model_np(d, latent, n_comp, centers_seed):
    rng = np.random.default_rng(centers_seed)
    W = rng.normal(0, 1, size=(d, latent)).astype(np.float32)
    comp = (2.0 * rng.normal(0, 1, size=(n_comp, latent))).astype(np.float32)
    w = 1.0 / np.arange(1, n_comp + 1)
    return W, comp, (w / w.sum())


def sift_hard(n, d=128, seed=1234, latent=16, n_comp=64, centers_seed=99):
    W, comp, w = _hard_model_np(d, latent, n_comp, centers_seed)
    rng = np.random.default_rng(seed)
    lab = rng.choice(n_comp, size=n, p=w)
    z = comp[lab] + rng.normal(0, 1, size=(n, latent)).astype(np.float32)
    x = 100.0 + 3.0 * (z @ W.T) + 4.0 * rng.normal(0, 1, size=(n, d)).astype(np.float32)
    return np.clip(np.rint(x), 0, 218).astype(np.float32)


def sift_hard_torch(n, d, seed, device, latent=16, n_comp=64, centers_seed=99, chunk=1 << 20):
    import torch
    gc = torch.Generator(device=device)
    gc.manual_seed(centers_seed)
    W = torch.randn((d, latent), generator=gc, device=device)
    comp = 2.0 * torch.randn((n_comp, latent), generator=gc, device=device)
    w = 1.0 / torch.arange(1, n_comp + 1, device=device, dtype=torch.float32)
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    out = torch.empty((n, d), dtype=torch.float32, device=device)
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        lab = torch.multinomial(w, e - s, replacement=True, generator=g)
        z = comp[lab] + torch.randn((e - s, latent), generator=g, device=device)
        x = 100.0 + 3.0 * (z @ W.T) + 4.0 * torch.randn((e - s, d), generator=g, device=device)
        out[s:e] = torch.clamp(torch.round(x), 0, 218)
    return out


def binary_clustered(n, d_bits, seed=1234, n_clusters=256, flip=0.1, centers_seed=99):
    """[n, d_bits / 8] uint8 packed binary rows (bit i at bit i & 7 of byte i >> 3): random centre bit vectors, each row
    a centre with every bit flipped independently at rate `flip`, so nearest neighbours share a centre and IVF recall
    is meaningful"""
    crng = np.random.default_rng(centers_seed)
    centres = crng.integers(0, 2, size=(n_clusters, d_bits), dtype=np.uint8)
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, n_clusters, size=n)
    bits = centres[lab] ^ (rng.random((n, d_bits)) < flip).astype(np.uint8)
    return np.packbits(bits, axis=1, bitorder="little")


def binary_clustered_torch(n, d_bits, seed, device, n_clusters=4096, flip=0.1, centers_seed=99, chunk=1 << 20):
    """binary_clustered generated on the device (another random stream): a torch uint8 [n, d_bits / 8] tensor"""
    import torch
    gc = torch.Generator(device=device)
    gc.manual_seed(centers_seed)
    centres = torch.randint(0, 2, (n_clusters, d_bits), generator=gc, device=device, dtype=torch.uint8)
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    weights = (2 ** torch.arange(8, device=device, dtype=torch.int32))
    out = torch.empty((n, d_bits // 8), dtype=torch.uint8, device=device)
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        lab = torch.randint(0, n_clusters, (e - s,), generator=g, device=device)
        flips = (torch.rand((e - s, d_bits), generator=g, device=device) < flip).to(torch.uint8)
        bits = (centres[lab] ^ flips).view(e - s, d_bits // 8, 8).to(torch.int32)
        out[s:e] = (bits * weights).sum(2).to(torch.uint8)
    return out
