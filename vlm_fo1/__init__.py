"""Drop-in mirror of the reference's ``vlm_fo1`` Python surface (om-ai-lab/VLM-FO1) over the H100 engine.

Same module paths, function names, signatures and return contracts as the reference (SURVEY.md section 8b), so the
reference's callers (``inference.py``, ``scripts/*.py``, ``evaluation/*.py``) import and run unmodified with this repo on
PYTHONPATH.  Nothing in here computes on the hot path: it builds ``generate()`` kwargs on the host and hands them to
``vlm-fo1_b200`` (libfo1.so)."""
