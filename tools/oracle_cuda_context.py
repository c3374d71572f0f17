"""Context number for the record (VERDICT r1 item 10; NOT a bench arm and not a parity check): the plain-PyTorch oracle of the same
forward run on torch-CUDA (cuDNN / cuBLAS) on the same GPU, with TF32 off (strict fp32 — the arithmetic class of this repo's f16s
engine) and TF32 on (what the reference executes on Ampere+ by default for convolutions).  B = 1, thinktwice.py config.

  python tools/oracle_cuda_context.py > gpurun_out/r2_oracle_cuda.json

The oracle's LiDAR voxelisation / rulebook code is host-side numpy, so when the full forward cannot run on the device the camera
encoder alone (93 % of the FLOPs) is timed and the line says so.
"""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def to_dev(x, dev):
    if torch.is_tensor(x):
        return x.to(dev)
    if isinstance(x, dict):
        return {k: to_dev(v, dev) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(to_dev(v, dev) for v in x)
    return x


def timed(fn, n=5):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    from oracle.model import EncoderDecoder as Oracle, init_oracle_weights
    from thinktwice_b200.config import Config, DEFAULT_CONFIG
    from thinktwice_b200.synthetic import make_batch
    cfg = Config.fromfile(DEFAULT_CONFIG)
    dev = torch.device('cuda:0')
    oracle = Oracle(**{k: v for k, v in cfg.model.items() if k != 'type'}).eval()
    init_oracle_weights(oracle, 0)
    ck = os.path.join(os.environ.get('TT_B200_CKPT_DIR', '/tmp'), 'tt_b200_synthetic_seed0.pth')
    if os.path.exists(ck):                                          # the bench's calibrated synthetic checkpoint, when present
        oracle.load_state_dict(torch.load(ck, map_location='cpu', weights_only=False)['state_dict'])
    oracle.to(dev)
    batch = make_batch(cfg, 1, seed=100)
    dbatch = {k: (to_dev(v, dev) if k != 'img_metas' else v) for k, v in batch.items()}
    res = {'what': 'plain-PyTorch oracle on torch-CUDA (cuDNN / cuBLAS), B = 1, thinktwice.py config; context only', 'torch': torch.__version__,
           'cudnn': torch.backends.cudnn.version()}
    with torch.no_grad():
        for tf32 in (False, True):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            torch.backends.cudnn.allow_tf32 = tf32
            key = 'tf32_on' if tf32 else 'tf32_off'
            try:
                ms = timed(lambda: oracle.forward_inference(dbatch))
                res[key] = {'scope': 'full forward (host-side voxelisation / rulebooks included)', 'ms_per_frame': ms, 'frames_per_s': 1000.0 / ms}
            except Exception as ex:                                     # noqa: BLE001 — context tool: report and fall back
                res[key + '_full_forward_error'] = repr(ex)[:300]
            try:
                ms = timed(lambda: oracle.img_encoder(dbatch['img'], batch['img_metas'], None))
                res[key + '_camera_encoder'] = {'scope': 'camera encoder only (A1-A8)', 'ms_per_frame': ms}
            except Exception as ex:                                     # noqa: BLE001
                res[key + '_camera_encoder_error'] = repr(ex)[:300]
    print(json.dumps(res))


if __name__ == '__main__':
    t0 = time.time()
    main()
