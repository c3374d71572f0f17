"""One rank of the two-process SyncBatchNorm check (tests/test_batch_norm_train_gpu.py): thinktwice_b200's SyncBatchNorm against
torch.nn.SyncBatchNorm in the same process, both over one gloo group on cuda:0.  Writes {case: max relative error} as JSON.

    python tests/batch_norm_sync_worker.py RANK WORLD STORE_FILE OUT_JSON
"""
import json
import os
import sys

import torch
import torch.distributed as dist
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from thinktwice_b200.ops import batch_norm as bn  # noqa: E402

# rows per rank: unequal, then one rank empty
CASES = {'unequal': (3, 2), 'empty_rank': (4, 0)}


def main():
    rank, world, store, out = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3], sys.argv[4]
    dist.init_process_group('gloo', init_method=f'file://{store}', rank=rank, world_size=world)
    res = {}
    try:
        for case, sizes in CASES.items():
            for relu, residual in ((False, False), (True, True)):
                torch.manual_seed(0)
                ref = nn.SyncBatchNorm(16, momentum=0.01).cuda()
                with torch.no_grad():
                    ref.weight.uniform_(0.5, 1.5)
                    ref.bias.uniform_(-0.5, 0.5)
                ours = bn.SyncBatchNorm(16, momentum=0.01).cuda()
                ours.load_state_dict(ref.state_dict())
                g = torch.Generator(device='cuda').manual_seed(10 + rank)
                shape = (sizes[rank], 16, 5, 7)
                x = (torch.randn(shape, generator=g, device='cuda') * 2 + 1).contiguous(memory_format=torch.channels_last)
                r = torch.randn(shape, generator=g, device='cuda') if residual else None
                gy = torch.randn(shape, generator=g, device='cuda')
                outs = []
                for m in (ref, ours):
                    xi = x.clone().requires_grad_(True)
                    ri = r.clone().requires_grad_(True) if residual else None
                    if m is ours:
                        y = m(xi, residual=ri, relu=relu)
                    else:
                        y = m(xi)
                        y = y + ri if residual else y
                        y = torch.relu(y) if relu else y
                    (y * gy).sum().backward()
                    outs.append(dict(y=y.detach(), grad_x=xi.grad, grad_r=ri.grad if residual else None, grad_w=m.weight.grad,
                                     grad_b=m.bias.grad, running_mean=m.running_mean, running_var=m.running_var,
                                     nbt=m.num_batches_tracked.float()))
                for k, a in outs[0].items():
                    if a is None or a.numel() == 0:
                        continue
                    err = float((outs[1][k] - a).abs().max() / a.abs().max().clamp_min(1e-12))
                    res[f'{case} relu={relu} residual={residual} {k}'] = err
    finally:
        dist.destroy_process_group()
    with open(out, 'w') as f:
        json.dump(res, f)


if __name__ == '__main__':
    main()
