"""CPU oracle for the b200bt hot path -- TEST INFRASTRUCTURE, not product code.

Everything under oracle/ is a CPU restatement of the reference's algorithm
(zd87pl/ai-crypto-trader @ 098e2ca), each function citing the reference
file:line it follows.  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference leg may import it, and only as the checker or
the timed CPU baseline.  The product package (ai_crypto_trader_b200) never
imports this package and has no CPU fallback.

Pinning status (see DESIGN.md "Oracle"):
  * simulate / metrics / advanced metrics / score / cross-validation / GA operators / Monte-Carlo statistics /
    StrategyTester backtest / portfolio VaR, CVaR and correlation are
    pinned by golden fixtures produced by EXECUTING the reference's own code
    (tests/golden/make_golden.py, run where a copy of the reference tree
    exists; fixtures committed under tests/golden/).
  * the `ta` indicator arithmetic is restated from the published definitions of
    the third-party `ta` package (unpinned `ta>=0.7.0`, requirements.txt:5; not
    vendored in the reference tree, not installed here): PARITY UNPINNED for
    that part -- it is cross-checked against pandas ewm/rolling only.
"""
