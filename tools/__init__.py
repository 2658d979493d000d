"""Developer tools: the OHEM oracle and golden generator, and the OHEM step benchmark.  Not part of the package."""
