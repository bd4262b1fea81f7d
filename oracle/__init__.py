"""CPU oracle for the DorPatch patch-generation hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``dorpatch_b200/`` may import this
package; only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs do, and only as the checker or the
timed CPU baseline -- never as the product path.

The oracle is a restatement (torch-CPU / numpy, fp32) of the reference
algorithm of the reference (CGCL-codes/DorPatch @ 0751fd4).  Each function
cites the reference file:line it follows.

Pinning status
--------------
* attack / defense arithmetic (attack.py, utils.py, defenses/PatchCleanser.py):
  PINNED -- checked against golden vectors produced by running the unmodified
  reference under a CPU shim (``oracle/ref_shim.py``; generator script
  ``tests/golden/make_golden.py``; vectors in ``tests/golden/*.npz``).
* classifier (timm==0.6.7 ``resnetv2_50x1_bit_distilled``): the architecture
  lives in a third-party dependency that is absent from the reference and
  from this image, and the reference holds no test that pins its outputs ->
  "parity unpinned" for the classifier itself.  The restatement in
  ``oracle/resnetv2.py`` is cross-checked layer-for-layer against the
  HuggingFace port ``transformers.models.bit`` (tests/test_oracle_resnetv2.py).
"""
