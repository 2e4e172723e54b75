"""Usage: python scratch/k2n_table_model.py GROUPS {balanced|firstfit} [r = scrambled keys]
CPU model of K2n's shared table (spgn_aggregate_kernel, bodo_b200/csrc/spgn.cuh) at the flagship shape: the keys of
bodo_b200/synth.py inserted one by one, in order of first appearance, with the kernel's spg_hash, spg_owner and spg_buckets,
132 owners (the SMs of an H100), and K2n's bucket slots.  Prints which keys live in their second bucket and which miss both
buckets (the stash, so the cold path on every one of their rows).  Sequential insertion: it does not model insert races."""
import numpy as np, sys

M64 = np.uint64((1 << 64) - 1)
def mix64(x):
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))

G = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
POLICY = sys.argv[2]
RANDOM = len(sys.argv) > 3
OWNERS = 132
NS = ((232448 - 256 - 9216) // 12 - 1024) & ~1  # max opt-in shared memory, static words, the warps' cold-row queues, stash
NB = NS // 2
seed = 1
n = 1 << 24
r = np.arange(0, n, dtype=np.uint64)
sk = np.uint64((seed * 0x9E3779B97F4A7C15) & ((1 << 64) - 1))
keys = (mix64(r ^ sk) % np.uint64(G)).astype(np.int64)
_, first = np.unique(keys, return_index=True)
order = keys[np.sort(first)]  # keys in order of first appearance
if RANDOM: order = (mix64(order.astype(np.uint64) + np.uint64(12345)) & np.uint64(0x7FFFFFFF)).astype(np.int64)
x = order.astype(np.uint64)
with np.errstate(over="ignore"):
    h = (x ^ (x >> np.uint64(29))) * np.uint64(0x9E3779B97F4A7C15)
hi32 = (h >> np.uint64(32)).astype(np.uint64)
owner = (hi32 * np.uint64(OWNERS)) >> np.uint64(32)
a1 = (h >> np.uint64(20)) & np.uint64(0xFFFFFFFF)
b1 = (a1 * np.uint64(NB)) >> np.uint64(32)
lo = h & np.uint64(0xFFFFFFFF)
t = (lo ^ ((h >> np.uint64(44)) & np.uint64(0xFFFFFFFF)))
t = (t * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)
b2 = (t * np.uint64(NB)) >> np.uint64(32)
b2 = np.where(b2 == b1, np.where(b1 + np.uint64(1) == np.uint64(NB), np.uint64(0), b1 + np.uint64(1)), b2)
stashed = np.zeros(len(order), bool); inb2 = np.zeros(len(order), bool)
per_owner = np.bincount(owner.astype(np.int64), minlength=OWNERS)
for o in range(OWNERS):
    idx = np.nonzero(owner == o)[0]
    fill = np.zeros(NB, np.int64)
    for i in idx:
        p, q = int(b1[i]), int(b2[i])
        f1, f2 = 2 - fill[p], 2 - fill[q]
        if f1 + f2 == 0:
            stashed[i] = True
            continue
        first_b = (q if f2 > f1 else p) if POLICY == 'balanced' else (p if f1 > 0 else q)
        if fill[first_b] < 2: fill[first_b] += 1; inb2[i] = first_b == q
        else:
            o2 = p if first_b == q else q; fill[o2] += 1; inb2[i] = o2 == q
frac = stashed.mean()
print(f"[{POLICY}{' random keys' if RANDOM else ' dense keys'}] groups {G}: keys per owner mean {per_owner.mean():.0f} max {per_owner.max()}, slot load {per_owner.mean()/NS:.3f}, "
      f"stashed keys {stashed.sum()} = {100*frac:.2f} % of keys (uniform keys: the same share of rows)")
for w in (32, 128):
    print(f"  P(a {w}-row warp iteration holds >= 1 cold row) = {1 - (1 - frac) ** w:.2f}")
fb2 = inb2.mean()
print(f"  keys living in their SECOND bucket: {100*fb2:.1f} %; P(a 32-lane warp row step has >= 1 such lane) = {1-(1-fb2)**32:.3f}")
