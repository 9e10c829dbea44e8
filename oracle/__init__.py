"""oracle/ -- TEST INFRASTRUCTURE, NOT PRODUCT.

CPU restatements (numpy / PyTorch-CPU) of the reference's stage-0 hot path, plus the recipe that
builds the reference's own CUDA extensions into oracle/_ref/ (build_ref.py).  Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this
package; nerf2mesh_b200/ never does.

Parity pinning status: the reference ships no tests, golden vectors or fixtures.  The oracle is
therefore pinned against outputs of the reference's OWN CUDA kernels (oracle/_ref, compiled
unmodified from the reference tree) committed under tests/golden/ together with the generating
script tests/golden/make_golden.py.
"""
