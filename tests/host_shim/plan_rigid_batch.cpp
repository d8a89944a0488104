// TEST INFRASTRUCTURE: plan_image.cpp's planner driver with PlanInput::replicaBodies set, built under this name by
// tests/test_batch_rigid_plan.py: a batch whose every replica has rigid bodies of its own (pbd_set_replica_rigid_bodies).
#include "host/image_plan.h"
namespace pbd_b200 {
static std::string plan_image_replica_bodies(const PlanInput &in, ImagePlan &out) {
    PlanInput with = in;
    with.replicaBodies = true;
    return plan_image(with, out);
}
}  // namespace pbd_b200
#define plan_image plan_image_replica_bodies
#include "plan_image.cpp"
