// TEST HELPER (not product code): blockdev_host.cpp's host build of the device-side block logic with its key-level part
// (blockdev_keylevel.inc) and the channel-capability entry points (blockdev_v13.inc).  Built as a library of its own.
#include "blockdev_host.cpp"
#include "blockdev_keylevel.inc"
#include "blockdev_v13.inc"
