import sys, numpy as np, torch
sys.path.insert(0, __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__))))
from torchio_b200 import ops
torch.manual_seed(0)
x = torch.rand(1, 1, 64, 64, 64, device='cuda')
mat = torch.tensor([[1, 0.05, 0, 0.5, -0.05, 1, 0, 1.0, 0, 0, 1, 0.25]], dtype=torch.float32, device='cuda')
hint = int(sys.argv[1]) if len(sys.argv) > 1 else 24
y = ops.resample(x, mat, None, None, (1, 1, 1), (1, 1, 1), affine_first=True, mode=1, fill=None, box_hint=hint)
torch.cuda.synchronize()
yr = ops.resample(x, mat, None, None, (1, 1, 1), (1, 1, 1), affine_first=True, mode=1, fill=None, box_hint=-1)
torch.cuda.synchronize()
print('max diff', float((y - yr).abs().max()))
