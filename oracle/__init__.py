"""CPU oracle for the Amphion vocoder-inference hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``amphion_b200/`` may import this
package: only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs are allowed to (see DESIGN.md §3).

The oracle is a restatement, in numpy / CPU-torch primitives, of the algorithm
in the reference files cited function by function.  It is pinned against
outputs of the reference modules themselves (``tests/golden/*.npz``, generated
by ``tests/golden/gen_golden.py`` which imports the reference (open-mmlab/Amphion)); the
reference ships no golden vectors or tests of its own for this path
(SURVEY.md §4), so those fixtures are the pin.
"""
from . import generator, mel  # noqa: F401
