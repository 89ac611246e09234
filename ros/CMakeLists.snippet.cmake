# Drop-in for object_tracking/CMakeLists.txt: replaces the three add_executable() blocks of the reference package.  The package
# keeps its own message definitions (msg/trackbox.msg, Obstacle.msg, ObstacleList.msg) and its package.xml; only the three node
# executables change.  LMOT_ROOT = a checkout of this repository with liblmot.so built (python -c "import __graft_entry__ as g; g.build()").
set(LMOT_ROOT "$ENV{LMOT_ROOT}" CACHE PATH "checkout of the H100 hot-path library")
set(LMOT_LIB ${LMOT_ROOT}/3d-lidar-multi-object-tracking_b200/liblmot.so)
foreach(node ground cluster tracking)
  add_executable(${node} ${LMOT_ROOT}/ros/src/${node}_node.cpp)
  target_include_directories(${node} PRIVATE ${LMOT_ROOT}/include ${LMOT_ROOT}/ros/include ${catkin_INCLUDE_DIRS})
  target_link_libraries(${node} ${catkin_LIBRARIES} ${LMOT_LIB})
  add_dependencies(${node} ${PROJECT_NAME}_generate_messages_cpp)
  set_target_properties(${node} PROPERTIES BUILD_RPATH ${LMOT_ROOT}/3d-lidar-multi-object-tracking_b200)
endforeach()
