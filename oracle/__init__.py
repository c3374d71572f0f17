"""CPU oracle for the ThinkTwice per-frame forward path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``thinktwice_b200/`` may import this
package; only ``tests/``, ``__graft_entry__.smoke()`` and the CPU-baseline /
``--impl reference`` legs of ``bench.py`` do, and there only as the checker or
the timed CPU baseline — never as the shipped path.

What it is: a plain-PyTorch fp32 restatement of the reference forward
(``/root/reference/open_loop_training``), module for module, with the same
``state_dict`` key names as the reference so that one set of weights drives both
the oracle and the H100 path.  The reference itself cannot be imported in this
image (mmcv / mmdet / mmdet3d / spconv are absent), so third-party pieces
(mmdet ResNet/PAFPN/BasicBlock, mmcv DCN / Voxelization / MSDA, mmdet3d
HardSimpleVFE / SparseEncoder / SECOND / SECONDFPN, spconv) are restated from
their published semantics; each function cites the reference call site it
follows.

PARITY STATUS.  The reference ships no tests, fixtures or golden vectors for this path (SURVEY.md §4, §8c), so the
pin comes from running the reference's own code:

(a) PINNED by the reference's own Python — tests/golden/make_reference_golden.py loads the in-tree files
    (encoder_decoder_framework.py, code/utils.py, model_code/backbones/lss.py, model_code/dense_heads/*) unmodified from
    /root/reference behind import stubs and runs them; tests/test_reference_golden_cpu.py checks this oracle against the
    stored outputs: BEV fusion + SE pyramid, the whole ThinkTwiceDecoder (B = 1 and the batch-coupled B = 2), the camera
    encoder LSS.forward at the plumbing shape (DepthNet / ASPP / UNet / seg->feature / PAFPN forward / frustum / geometry
    / lift / sweeps), EncoderDecoder.forward_inference end to end at the plumbing shape, process_action / control_pid —
    bit-exact, and the state_dict names and shapes identical.
(b) PINNED by the reference's own CUDA kernel — voxel pooling, compiled from /root/reference into ``oracle/_ref``
    (oracle/build_ref.py) and run beside the product kernel on the GPU box.
(c) UNPINNED (third-party code that is not under /root/reference; restated from published semantics and held by
    self-checks against independent formulations, tests/test_oracle_selfcheck.py): mmdet ResNet-50 (== torchvision trunk)
    and PAFPN/BasicBlock layer construction, mmcv DCN (== torchvision deform_conv2d; zero offset == grouped conv),
    mmcv multi_scale_deformable_attn_pytorch (== brute-force bilinear loops), and the whole LiDAR branch — mmcv
    Voxelization, mmdet3d HardSimpleVFE / SparseEncoder / SECOND / SECONDFPN, spconv (sparse conv == masked dense conv3d).
    In (a) these leaves are the oracle's own restatements on both sides.
(d) committed golden vectors the oracle generated itself (tests/golden/make_golden.py) carry it to the GPU tests.
"""
