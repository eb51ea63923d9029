// solver2d-b200 — s2World_Draw: the read-back path of the samples harness (behaviour of reference src/world.c:308-563,
// src/joint.c:467-505, src/revolute_joint.c:890-984). It is the one API call that needs *everything* back on the host:
// body transforms (lazy sync), shape boxes (when AABBs are drawn) and the contact table (when contact points are
// drawn). Nothing here is on the step path.
#include "s2_host.h"
#include "shared/s2_collide.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>

static s2Color s2Rgb(float r, float g, float b)
{
	s2Color c = {r, g, b, 1.0f};
	return c;
}

static void s2DrawShape(s2DebugDraw* draw, const s2Shape* shape, s2Transform xf, s2Color color)
{
	switch (shape->type)
	{
		case s2_capsuleShape:
			draw->DrawSolidCapsule(s2TransformPoint(xf, shape->capsule.point1), s2TransformPoint(xf, shape->capsule.point2),
								   shape->capsule.radius, color, draw->context);
			break;

		case s2_circleShape:
			draw->DrawSolidCircle(s2TransformPoint(xf, shape->circle.point), shape->circle.radius,
								  s2RotateVector(xf.q, s2MakeVec2(1.0f, 0.0f)), color, draw->context);
			break;

		case s2_polygonShape:
		{
			const s2Polygon* poly = &shape->polygon;
			s2Vec2 vertices[s2_maxPolygonVertices];
			for (int i = 0; i < poly->count; ++i)
			{
				vertices[i] = s2TransformPoint(xf, poly->vertices[i]);
			}
			if (poly->radius > 0.0f)
			{
				s2Color fill = {0.5f * color.r, 0.5f * color.g, 0.5f * color.b, 0.5f};
				draw->DrawRoundedPolygon(vertices, poly->count, poly->radius, fill, color, draw->context);
			}
			else
			{
				draw->DrawSolidPolygon(vertices, poly->count, color, draw->context);
			}
		}
		break;

		case s2_segmentShape:
			draw->DrawSegment(s2TransformPoint(xf, shape->segment.point1), s2TransformPoint(xf, shape->segment.point2), color,
							  draw->context);
			break;

		default:
			break;
	}
}

static void s2DrawJoint(s2DebugDraw* draw, s2World* world, const s2Joint* joint)
{
	const s2Body* bodyA = world->bodies + joint->bodyIndexA;
	const s2Body* bodyB = world->bodies + joint->bodyIndexB;
	s2Transform xfA = {bodyA->origin, bodyA->rot};
	s2Transform xfB = {bodyB->origin, bodyB->rot};
	s2Vec2 pA = s2TransformPoint(xfA, joint->localOriginAnchorA);
	s2Vec2 pB = s2TransformPoint(xfB, joint->localOriginAnchorB);

	if (joint->type == s2_mouseJoint)
	{
		s2Color green = s2Rgb(0.0f, 1.0f, 0.0f);
		draw->DrawPoint(joint->targetA, 4.0f, green, draw->context);
		draw->DrawPoint(pB, 4.0f, green, draw->context);
		draw->DrawSegment(joint->targetA, pB, s2Rgb(0.8f, 0.8f, 0.8f), draw->context);
		return;
	}

	draw->DrawPoint(pA, 5.0f, s2Rgb(0.3f, 0.3f, 0.9f), draw->context);
	draw->DrawPoint(pB, 5.0f, s2Rgb(0.4f, 0.4f, 0.4f), draw->context);

	if (joint->type == s2_motorJoint)
	{
		// the segment from the target point (A's linear offset) to B's origin: the pose error the motor is removing
		draw->DrawSegment(pA, pB, s2Rgb(0.8f, 0.5f, 0.9f), draw->context);
		return;
	}

	if (joint->type == s2_pulleyJoint)
	{
		// Box2D 2.4's three segments: each rope from its ground anchor to its body anchor, and the line between the ground
		// anchors
		s2Color color = s2Rgb(0.5f, 0.8f, 0.8f);
		draw->DrawSegment(joint->targetA, pA, color, draw->context);
		draw->DrawSegment(joint->localAxisA, pB, color, draw->context);
		draw->DrawSegment(joint->targetA, joint->localAxisA, color, draw->context);
		return;
	}

	if (joint->type == s2_gearJoint)
	{
		// Box2D 2.4's default joint lines: each body's origin to its anchor, and anchor A to anchor B
		s2Color color = s2Rgb(0.5f, 0.8f, 0.8f);
		draw->DrawSegment(xfA.p, pA, color, draw->context);
		draw->DrawSegment(pA, pB, color, draw->context);
		draw->DrawSegment(xfB.p, pB, color, draw->context);
		return;
	}

	if (joint->type == s2_distanceJoint)
	{
		// the segment between the anchors and, with the limit on, a mark across the line at minLength and at maxLength from
		// anchor A
		draw->DrawSegment(pA, pB, s2Rgb(0.5f, 0.8f, 0.8f), draw->context);
		if (joint->enableLimit)
		{
			float length;
			s2Vec2 axis = s2cGetLengthAndNormalize(&length, s2Sub(pB, pA));
			s2Vec2 perp = s2MulSV(0.5f * joint->drawSize, s2LeftPerp(axis));
			s2Vec2 lower = s2MulAdd(pA, joint->lowerAngle, axis);
			s2Vec2 upper = s2MulAdd(pA, joint->upperAngle, axis);
			draw->DrawSegment(s2Sub(lower, perp), s2Add(lower, perp), s2Rgb(0.3f, 0.9f, 0.3f), draw->context);
			draw->DrawSegment(s2Sub(upper, perp), s2Add(upper, perp), s2Rgb(0.9f, 0.3f, 0.3f), draw->context);
		}
		return;
	}

	if (joint->type == s2_prismaticJoint || joint->type == s2_wheelJoint)
	{
		// the axis through anchor A (drawSize each way), a mark across the axis at each translation limit, and the
		// segment from anchor A to anchor B; the same for a wheel joint
		const float L = joint->drawSize;
		s2Vec2 axis = s2RotateVector(bodyA->rot, joint->localAxisA);
		s2Vec2 perp = s2MulSV(0.5f * L, s2LeftPerp(axis));
		draw->DrawSegment(s2MulSub(pA, L, axis), s2MulAdd(pA, L, axis), s2Rgb(0.7f, 0.7f, 0.7f), draw->context);
		if (joint->enableLimit)
		{
			s2Vec2 lower = s2MulAdd(pA, joint->lowerAngle, axis);
			s2Vec2 upper = s2MulAdd(pA, joint->upperAngle, axis);
			draw->DrawSegment(s2Sub(lower, perp), s2Add(lower, perp), s2Rgb(0.3f, 0.9f, 0.3f), draw->context);
			draw->DrawSegment(s2Sub(upper, perp), s2Add(upper, perp), s2Rgb(0.9f, 0.3f, 0.3f), draw->context);
		}
		draw->DrawSegment(pA, pB, s2Rgb(0.5f, 0.8f, 0.8f), draw->context);
		return;
	}

	const float L = joint->drawSize;
	s2Color grey = s2Rgb(0.7f, 0.7f, 0.7f);
	s2Vec2 r = s2RotateVector(bodyB->rot, s2MakeVec2(L * cosf(joint->referenceAngle), L * sinf(joint->referenceAngle)));
	draw->DrawSegment(pB, s2Add(pB, r), grey, draw->context);
	draw->DrawCircle(pB, L, grey, draw->context);

	if (joint->enableLimit)
	{
		s2Vec2 rlo = s2RotateVector(bodyA->rot, s2MakeVec2(L * cosf(joint->lowerAngle), L * sinf(joint->lowerAngle)));
		s2Vec2 rhi = s2RotateVector(bodyA->rot, s2MakeVec2(L * cosf(joint->upperAngle), L * sinf(joint->upperAngle)));
		draw->DrawSegment(pB, s2Add(pB, rlo), s2Rgb(0.3f, 0.9f, 0.3f), draw->context);
		draw->DrawSegment(pB, s2Add(pB, rhi), s2Rgb(0.9f, 0.3f, 0.3f), draw->context);
	}

	s2Color link = s2Rgb(0.5f, 0.8f, 0.8f);
	draw->DrawSegment(xfA.p, pA, link, draw->context);
	draw->DrawSegment(pA, pB, link, draw->context);
	draw->DrawSegment(xfB.p, pB, link, draw->context);
}

void s2World_Draw(s2WorldId worldId, s2DebugDraw* draw)
{
	s2World* world = s2GetWorldFromId(worldId);
	s2SyncStateToHost(world);
	char buffer[32];

	if (draw->drawShapes)
	{
		for (int i = 0; i < world->bodyPool.capacity; ++i)
		{
			const s2Body* body = world->bodies + i;
			if (s2IsFree(&body->object))
			{
				continue;
			}
			s2Transform xf = {body->origin, body->rot};
			s2Color color = draw->dynamicBodyColor;
			if (body->type == s2_dynamicBody && body->mass == 0.0f)
			{
				color = s2Rgb(0.9f, 0.1f, 0.1f); // dynamic body without mass
			}
			else if (body->type == s2_staticBody)
			{
				color = s2Rgb(0.5f, 0.9f, 0.5f);
			}
			else if (body->type == s2_kinematicBody)
			{
				color = s2Rgb(0.5f, 0.5f, 0.9f);
			}
			for (int si = body->shapeList; si != S2_NULL_INDEX; si = world->shapes[si].nextShapeIndex)
			{
				s2DrawShape(draw, world->shapes + si, xf, color);
			}
		}
	}

	if (draw->drawJoints)
	{
		for (int i = 0; i < world->jointPool.capacity; ++i)
		{
			const s2Joint* joint = world->joints + i;
			if (s2ObjectValid(&joint->object))
			{
				s2DrawJoint(draw, world, joint);
			}
		}
	}

	if (draw->drawAABBs)
	{
		s2SyncBoxesToHost(world);
		s2Color color = s2Rgb(0.9f, 0.3f, 0.9f);
		for (int i = 0; i < world->bodyPool.capacity; ++i)
		{
			const s2Body* body = world->bodies + i;
			if (s2IsFree(&body->object))
			{
				continue;
			}
			snprintf(buffer, sizeof(buffer), "%d", body->object.index);
			draw->DrawString(body->position, buffer, draw->context);
			for (int si = body->shapeList; si != S2_NULL_INDEX; si = world->shapes[si].nextShapeIndex)
			{
				s2Box box = world->shapes[si].fatAABB;
				s2Vec2 vs[4] = {{box.lowerBound.x, box.lowerBound.y},
								{box.upperBound.x, box.lowerBound.y},
								{box.upperBound.x, box.upperBound.y},
								{box.lowerBound.x, box.upperBound.y}};
				draw->DrawPolygon(vs, 4, color, draw->context);
			}
		}
	}

	if (draw->drawMass)
	{
		for (int i = 0; i < world->bodyPool.capacity; ++i)
		{
			const s2Body* body = world->bodies + i;
			if (s2IsFree(&body->object))
			{
				continue;
			}
			s2Transform xf = {body->position, body->rot};
			draw->DrawTransform(xf, draw->context);
			snprintf(buffer, sizeof(buffer), "%.2g", body->mass);
			draw->DrawString(body->position, buffer, draw->context);
		}
	}

	if (draw->drawContactPoints)
	{
		s2bCounters counters;
		s2b_get_counters(world->device, &counters);
		int n = counters.contactCount;
		s2bContactRow* rows = (s2bContactRow*)malloc(sizeof(s2bContactRow) * (size_t)(n > 0 ? n : 1));
		n = s2b_download_contacts(world->device, rows, n);
		for (int i = 0; i < n; ++i)
		{
			const s2bContactRow* c = rows + i;
			s2Vec2 normal = {c->normal[0], c->normal[1]};
			const s2Body* bodyA = world->bodies + c->bodyA;
			s2Transform xfA = {bodyA->origin, bodyA->rot};
			for (int j = 0; j < c->pointCount; ++j)
			{
				const s2bContactPoint* point = c->points + j;
				s2Vec2 worldPoint = s2TransformPoint(xfA, s2MakeVec2(point->localAnchorA[0], point->localAnchorA[1]));
				if (point->separation > s2_linearSlop)
				{
					draw->DrawPoint(worldPoint, 5.0f, s2Rgb(0.3f, 0.3f, 0.3f), draw->context); // speculative
				}
				else if (point->persisted == 0)
				{
					draw->DrawPoint(worldPoint, 10.0f, s2Rgb(0.3f, 0.95f, 0.3f), draw->context); // added this step
				}
				else
				{
					draw->DrawPoint(worldPoint, 5.0f, s2Rgb(0.3f, 0.3f, 0.95f), draw->context); // persisted
				}

				if (draw->drawContactNormals)
				{
					draw->DrawSegment(worldPoint, s2MulAdd(worldPoint, 0.3f, normal), s2Rgb(0.9f, 0.9f, 0.9f), draw->context);
				}
				else if (draw->drawContactImpulses)
				{
					draw->DrawSegment(worldPoint, s2MulAdd(worldPoint, point->normalImpulse, normal), s2Rgb(0.9f, 0.9f, 0.3f),
									  draw->context);
					snprintf(buffer, sizeof(buffer), "%.2g", point->normalImpulse);
					draw->DrawString(worldPoint, buffer, draw->context);
				}

				if (draw->drawFrictionImpulses)
				{
					s2Vec2 tangent = s2RightPerp(normal);
					draw->DrawSegment(worldPoint, s2MulAdd(worldPoint, point->tangentImpulse, tangent), s2Rgb(0.9f, 0.9f, 0.3f),
									  draw->context);
					snprintf(buffer, sizeof(buffer), "%.2g", point->normalImpulse);
					draw->DrawString(worldPoint, buffer, draw->context);
				}
			}
		}
		free(rows);
	}
}
