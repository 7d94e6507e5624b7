# Builds the pose-interpolation oracle (orc_pose.c) on its own; same flags as oracle/Makefile (the reference's
# Release defaults, -ffp-contract=off pins "no FMA").  orc_align.c is compiled in for its orc_posev_exp, so PoseV::exp
# has one definition.  Test infrastructure only.
CC := /usr/bin/gcc
CFLAGS = -O3 -DNDEBUG -std=c11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

all: libouster_oracle_pose.so

libouster_oracle_pose.so: orc_pose.c orc_align.c
	$(CC) $(CFLAGS) -shared -o $@ orc_pose.c orc_align.c -lm

clean:
	rm -f libouster_oracle_pose.so
