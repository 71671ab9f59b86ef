"""Plain-integer restatement of the device draw of xunet_srn_batch (csrc/data.cu): the Feistel permutation of one epoch, the
target view and the per-micro-batch diffusion seed.  Written independently of srn_data's vectorised numpy version, one draw at
a time, so the two can be checked against each other."""
M64 = (1 << 64) - 1


def mix64(z: int) -> int:
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def permute(x: int, n: int, seed: int, epoch: int) -> int:
    h = 1
    while 4 ** h < n:
        h += 1
    mask = (1 << h) - 1
    base = mix64(seed ^ 0x243F6A8885A308D3)
    keys = [mix64(base + 4 * epoch + r) for r in range(4)]
    while True:
        left, right = x >> h, x & mask
        for k in keys:
            left, right = right, left ^ (mix64(right ^ k) & mask)
        x = (left << h) | right
        if x < n:
            return x


def draw(first, count, item_inst, seed: int, c: int, j: int, k: int, rank: int, world: int, B: int, b: int):
    """(inst, v, v2) of sample b."""
    n = len(item_inst)
    g = (((c * k + j) * world + rank) * B + b) & M64
    item = permute(g % n, n, seed, g // n)
    inst = int(item_inst[item])
    v2 = mix64(mix64(seed ^ 0x13198A2E03707344) + g) % int(count[inst])
    return inst, item - int(first[inst]), v2


def diffusion_seed(seed: int, c: int, j: int, k: int, rank: int) -> int:
    return mix64(mix64(mix64(seed ^ 0xA4093822299F31D0) + c * k + j) + rank)
