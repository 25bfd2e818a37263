"""Sequential recommenders on the time-ordered samplers: FPMC and TransRec (high_order = 1), HRM, NPE and FPMCplus (a
window of high_order recent items), Caser (convolutions over the last seq_L items)."""
