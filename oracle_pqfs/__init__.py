"""IVFPQFastScan CPU restatement: a C library (ivfpqfs_oracle.c via ivfpqfs.py) and its numpy twin (twin.py).
Test infrastructure only; the product package never imports it."""
