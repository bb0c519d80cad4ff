import sys; sys.path.insert(0, __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__))))
import torch
from torchio_b200 import ops
for seed, offset, n in [(0, 0, 16), (1234, 0, 64), (1234, 0, 4096), (7, 0, 3 * 2**20 + 1600), (99, 40 * 2**20, 2**21 + 32)]:
    g = torch.Generator().manual_seed(seed)
    if offset:
        torch.randn(offset, generator=g)
    want = torch.randn(n, generator=g)
    got = ops.randn_mt19937(seed, offset, n, "cuda").cpu()
    d = (got - want).abs()
    bad = (d > 2e-6).nonzero().flatten()
    print(seed, offset, n, 'max', float(d.max()), 'nbad', bad.numel(), 'first bad', bad[:5].tolist(), 'frac bit-identical', float((got == want).float().mean()))
    if bad.numel():
        i = int(bad[0]); print('  got', got[i-2:i+3].tolist(), 'want', want[i-2:i+3].tolist())
