// TEST INFRASTRUCTURE: the planner driver of plan_image.cpp, built under this name by tests/test_batch_plan.py.  Its input starts with the
// size of the replica batch, so one driver serves single scenes and batches.
#include "plan_image.cpp"
