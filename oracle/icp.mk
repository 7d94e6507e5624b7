# Builds the frame-to-map registration oracle (orc_icp.c) on its own; same flags as oracle/Makefile (the reference's
# Release defaults, -ffp-contract=off pins "no FMA").  Test infrastructure only.
CC := /usr/bin/gcc
CFLAGS = -O3 -DNDEBUG -std=c11 -fPIC -ffp-contract=off -Wall -Wextra -Wno-unused-parameter

all: libouster_oracle_icp.so

libouster_oracle_icp.so: orc_icp.c
	$(CC) $(CFLAGS) -shared -o $@ orc_icp.c -lm

clean:
	rm -f libouster_oracle_icp.so
