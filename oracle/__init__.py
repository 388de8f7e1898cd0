"""CPU oracle for the DiffSensei UNet sampling path — TEST INFRASTRUCTURE ONLY.

This package is a plain-PyTorch (CPU, fp32) restatement of the arithmetic on the reference's hot
path (SURVEY.md §8a).  It exists so that the sm_90a kernels in ``diffsensei_b200`` can be checked
against the reference's results.  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import it; the product package
``diffsensei_b200`` never does (tests/test_no_oracle_leak.py enforces this).

Parity pinning (SURVEY.md §8c): the reference ships no tests, golden vectors or fixtures, and
``diffusers`` (which holds ~85 % of the arithmetic) is neither vendored nor installed here.
  * ``oracle.attention`` and ``oracle.resampler`` restate ``src/models/attention_processor.py`` and
    ``src/models/resampler.py``.  Those two reference files import only torch, so they WERE executed in
    the build container; their outputs on seeded inputs are committed under ``tests/golden/`` by
    ``tools/make_golden.py`` and the restatement is pinned to them  -> pinned.
  * ``oracle.unet`` (diffusers SDXL blocks) and ``oracle.ddim`` restate published diffusers behaviour
    from its documented semantics; no reference output exists to pin them  -> **parity unpinned** for
    those blocks (stated in DESIGN.md).
"""
