"""What more than one test module shares: fp64 references, error budgets, scene builders and the record files.

No module here starts with test_, so pytest does not collect them, and none imports a test module.  Importing one
runs no CUDA, builds no tree and reads no golden file: that work happens inside the functions.
"""
