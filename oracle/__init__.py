"""CPU oracle for the hydragnn-b200 hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``hydragnn_b200/`` imports this
package; the only permitted importers are ``tests/``, ``__graft_entry__.smoke()``
and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs.  The product
path fails loudly when its CUDA library is missing instead of falling back here.

Every function is a pure-torch / numpy restatement of one reference function and
cites the reference ``file:line`` it follows (paths relative to the reference
checkout of ORNL/HydraGNN @ 6c45f168).

Parity pin status (see DESIGN.md "Oracle"):

* EGNN ``E_GCL``, PaiNN ``PainnMessage`` / ``PainnUpdate``, ``sinc_expansion``,
  ``cosine_cutoff``, ``get_edge_vectors_and_lengths``, ``unsorted_segment_mean``,
  ``MLPNode``, the MLIP ``energy_force_loss`` arithmetic and the NumPy
  post-processing of ``RadiusGraphPBC`` are PINNED: ``tests/golden/*.pt`` were
  produced by importing the reference's own modules (third-party imports that
  are absent from this image stubbed out, see ``tests/golden/make_golden.py``).
* ``radius_graph`` (torch_cluster 1.6.3) and the raw vesin 0.4.2 neighbour list
  are restated from the published algorithms; the reference's known-answer PBC
  tests (H2: 1/2 neighbours, BCC Cr 5x5x5: 14/15) and the rotational-invariance
  test pin counts and edge sets.  Ordering under ``max_neighbours`` truncation
  is "parity unpinned" (no golden vectors exist in the reference).
* The PNA, PNAPlus, CGCNN, GAT and SchNet stacks (``pna``, ``pnaplus``, ``cgcnn``, ``gat``,
  ``schnet``) are PINNED by ``tests/golden/models_{pna,pnaplus,cgcnn,gat,schnet}.pt``,
  produced by the reference's own stack, ``Base.py`` and ``gps.py`` with the PyG convs
  restated here standing in for PyG's; each restated conv is pinned by hand-computed
  cases in ``tests/test_oracle_*.py``.
* The GaussianNLLLoss mean-and-variance heads and the shared PReLU slope of every
  stack (``base.StackOracle``), and MACE's edge attributes and graph-attribute
  conditioning (``mace.MACEOracle``), are PINNED by
  ``tests/golden/models_{gnll,prelu,mace_edge,mace_cond}.pt``, produced by the
  reference's own ``Base.py``, stacks and MACE blocks.
"""

from . import geometry, radius_graph, egnn, painn, base, mlip  # noqa: F401
