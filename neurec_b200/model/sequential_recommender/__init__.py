"""Sequential recommenders on the time-ordered samplers: FPMC and TransRec (high_order = 1), HRM, NPE and FPMCplus (a
window of high_order recent items)."""
