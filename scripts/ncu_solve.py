"""One solve of a small cfg2 batch (for an ncu capture of the persistent solve_kernel)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from trajopt_b200 import api, problems
B = int(sys.argv[1]) if len(sys.argv) > 1 else 132  # one trajectory per SM of an H100 SXM
d = problems.config2(B=B, T=30)
p = api.Problem(d)
got = p.solve()
print("solved", B, "converged", int((got["status"] == 0).sum()), "gpu ms", got["timing"]["total_ms"])
