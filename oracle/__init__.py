"""CPU parity oracle for the OccDepth forward hot path.  TEST INFRASTRUCTURE ONLY.

Nothing under `occdepth_b200/` may import this package; only `tests/`, `__graft_entry__.smoke()` and
`bench.py`'s CPU-baseline legs do.  Contents:

* `functional.py`  plain-PyTorch fp32 restatement (state_dict-driven, functional style) of every reference
                   function on the hot path, each citing the reference file:line it follows
* `projection.py`  numpy restatement of the data pipeline's voxel -> pixel projection (`vox2pix`), pinned bit for bit
                   against the reference's numba implementation
* `effnet.py`      geffnet-shaped `tf_efficientnet_b*_ns` definition (the reference fetches it with
                   torch.hub at run time; un-vendored, see DESIGN.md "oracle")
* `synth.py`       re-export of /synthetic.py: seeded synthetic inputs / weights / `vox2pix` restatement (SURVEY 8d)
* `ref_import.py`  imports the UNMODIFIED reference from a checkout of the original project ($OCCDEPTH_REFERENCE)
                   behind `shims/`; used to generate `tests/golden/*`
* `gen_golden.py`  the script that generated `tests/golden/*.pt`

Pinning status: the reference ships no tests or golden vectors.  `functional.py` is pinned against the
reference's own modules executed on CPU: tests/test_oracle_vs_reference.py, tests/test_golden.py and
tests/test_state_dict_compat.py compare with the fixtures those runs produced (tests/golden/).
The EfficientNet encoder is the exception: geffnet is not in the original project nor installable offline, so
`effnet.py` is pinned only against torchvision's independent EfficientNet (same weights, odd input sizes
where TF-SAME == symmetric padding) -- "parity unpinned" w.r.t. geffnet itself.
"""
