"""GPU: the device field and scalar primitives (PTX limb arithmetic, the in-place and paired multipliers, the division-step
inversions) against Python integers, through the op table of fabric-mod_b200/csrc/fieldops.cuh.  tests/test_host_sim.py checks the
host build of the same table with the same expectations (util.field_op_cases)."""
import random

import numpy as np
import pytest

from util import be32, field_op_cases, from_be, pkg

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = pkg().binding.Context(max_batch=4096)
    yield c
    c.close()


def test_field_primitives(ctx):
    """Every op: 4000 random operands plus every pair of edge operands (0, 1, m - 1, m - 2, 2^255, 2^224, 2^256 - 1 ...) for the
    products, sums and differences; 4000 random units plus small and structured values for the inversions.  The products run through
    fe_mul / fe_sqr (out of line), fe_mul2 (either output, with a different product in the other slot), and the forms expanded in
    place that the key-table and small-table kernels use (fe_mul_t / fe_sqr_t / fe_mul2_t with INL = true)."""
    for op, (a, b, exp) in field_op_cases(random.Random(1), 4000).items():
        A = np.stack([be32(x) for x in a]); B = np.stack([be32(x) for x in b])
        assert [from_be(row) for row in ctx.test_fieldop(op, A, B)] == exp, op


def test_unknown_op_is_refused(ctx):
    z = np.zeros((1, 32), np.uint8)
    for op in (-1, 17):
        with pytest.raises(pkg().binding.FabGpuError):
            ctx.test_fieldop(op, z, z)
